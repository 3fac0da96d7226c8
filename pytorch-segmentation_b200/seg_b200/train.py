"""Fused training step for the engine models: forward -> fused upsample (or pixel shuffle) + CE (no full-resolution
logits in HBM) -> backward -> (NCCL gradient all-reduce) -> fused multi-tensor SGD.  Same arithmetic as one iteration of the
reference's Trainer._train_epoch (trainer.py:55-71) with torch.optim.SGD and differential learning rates
(base/base_trainer.py:46-57), minus the host synchronisations.  Optionally also the training metrics of trainer.py:84-86
and the validation pass of Trainer._valid_epoch (trainer.py:109-165), from the same fused loss kernel.
"""
import numpy as np
import torch
import torch.distributed as dist

from . import lib
from . import metrics as _metrics
from .engine import Tape


class WeightTables:
    """Persistent packed-weight (bf16) and packed-weight-gradient (fp32) buffers for every dense conv of a model, plus the
    device tables that let ONE launch pack all weights / unpack all weight gradients (instead of 2 x ~114 small
    launches).  Shared by `FusedTrainStep` and the graph-replayed plugin path (`nets._GraphEntry`).

    grad_views: Parameter -> fp32 gradient tensor in the parameter's OIHW layout (where `unpack()` writes); None =
    forward only."""

    def __init__(self, model, grad_views, dev):
        specs = [s for s in model.all_conv_specs()]
        self.specs = specs
        for ds in model.all_dw_specs():
            ds.always_repack = True  # in-place optimiser kernels / graph replays do not go through the version check
        dt = np.dtype([("oihw", "<u8"), ("packed", "<u8"), ("K", "<i4"), ("C", "<i4"), ("R", "<i4"), ("S", "<i4"),
                       ("Cpad", "<i4"), ("explicit", "<i4"), ("start", "<i8")])
        assert dt.itemsize == lib.load().seg_pack_entry_bytes()
        want_g = grad_views is not None  # forward-only users (validation graphs) need no gradient accumulators
        n_dw = sum(int(np.prod(s.packed_shape())) for s in specs if s.m.weight.requires_grad) if want_g else 0
        self.flat_dwp = torch.zeros(n_dw, dtype=torch.float32, device=dev)
        pack = np.zeros(len(specs), dtype=dt)
        unp = []
        self.packed_bufs, self.dw_bufs = {}, {}
        p_start = u_start = off = 0
        for i, s in enumerate(specs):
            shape = s.packed_shape()
            buf = torch.empty(shape, dtype=torch.bfloat16, device=dev)
            self.packed_bufs[s] = buf
            w = s.m.weight
            pack[i] = (w.data_ptr(), buf.data_ptr(), s.K, s.C, s.R, s.S, shape[2], int(s.explicit), p_start)
            p_start += int(np.prod(shape))
            if want_g and w.requires_grad:
                n = int(np.prod(shape))
                dwb = self.flat_dwp[off:off + n].view(shape)
                self.dw_bufs[s] = dwb
                off += n
                unp.append((grad_views[w].data_ptr(), dwb.data_ptr(), s.K, s.C, s.R, s.S, shape[2], int(s.explicit), u_start))
                u_start += w.numel()
        self.pack_total, self.unpack_total = p_start, u_start
        self.pack_table = torch.from_numpy(pack.view(np.uint8).copy()).to(dev)
        self.unpack_n = len(unp)
        self.unpack_table = torch.from_numpy(np.array(unp, dtype=dt).view(np.uint8).copy()).to(dev) if unp else None
        self._unp, self._unp_params, self._dt, self._dev = unp, [s.m.weight for s in specs if (want_g and s.m.weight.requires_grad)], dt, dev
        self.param_ptrs = [s.m.weight.data_ptr() for s in specs]

    def unpack_subtables(self, bucket_of):
        """One unpack table per gradient bucket (bucket_of: Parameter -> bucket id): list of (device table, n, total) so a
        bucket's packed weight gradients can be unpacked — and its all-reduce launched — as soon as its last wgrad retired."""
        groups = {}
        for entry, p in zip(self._unp, self._unp_params):
            groups.setdefault(bucket_of[p], []).append(entry)
        out = {}
        for b, entries in groups.items():
            start, fixed = 0, []
            for e in entries:
                fixed.append(e[:8] + (start,))
                start += e[2] * e[3] * e[4] * e[5]  # K*C*R*S elements of the OIHW gradient
            out[b] = (torch.from_numpy(np.array(fixed, dtype=self._dt).view(np.uint8).copy()).to(self._dev), len(fixed), start)
        return out

    def stale(self):
        """True when a parameter was re-allocated (e.g. model.to(...), load_state_dict on a fresh module): the tables
        hold raw pointers."""
        return any(s.m.weight.data_ptr() != q for s, q in zip(self.specs, self.param_ptrs))

    def pack(self):
        lib.call("seg_pack_weights_batched", self.pack_table.data_ptr(), len(self.specs), self.pack_total)

    def zero_wgrads(self):
        self.flat_dwp.zero_()

    def unpack(self):
        if self.unpack_n:
            lib.call("seg_unpack_wgrads_batched", self.unpack_table.data_ptr(), self.unpack_n, self.unpack_total, 0.0)


def _loss_spec(loss, ignore_index):
    """(ignore_index, LossSpec) for FusedTrainStep's `loss`; None is the unweighted mean cross-entropy."""
    from . import losses
    if loss is None:
        return (255 if ignore_index is None else ignore_index), losses.LossSpec(None, None, True)
    if type(loss) not in (losses.CrossEntropyLoss2d, losses.FocalLoss):
        raise NotImplementedError(
            f"FusedTrainStep fuses seg_b200.CrossEntropyLoss2d and seg_b200.FocalLoss only, not {type(loss).__name__}; "
            "train with it on the plugin surface instead: loss = crit(model(x), y); loss.backward(); optimizer.step()")
    if ignore_index is not None and ignore_index != loss.ignore_index:
        raise ValueError(f"FusedTrainStep: ignore_index={ignore_index} conflicts with the loss's ignore_index={loss.ignore_index}")
    return loss.ignore_index, loss.spec


class FusedTrainStep:
    """loss: None (the reference configs' CrossEntropyLoss2d(ignore_index=255)), or a seg_b200.CrossEntropyLoss2d /
    seg_b200.FocalLoss instance, applied to the main head and (x aux_weight) to the aux head; its ignore_index governs.

    metrics=True: every step() and evaluate() adds the main head's eval_metrics counters (trainer.py:62,84) into the
    device vector `seg_counters` (int64 [2 + 3C]: correct, labeled, inter[C], pred[C], lab[C]) inside the fused loss
    launch, so graph replays count too; `seg_metrics()` turns the running totals into Trainer._get_seg_metrics's dict and
    `reset_metrics()` zeroes them."""

    EVAL_GRAPHS_MAX = 2  # evaluate() input shapes captured at most (the batch and a smaller last batch); others run eagerly

    def __init__(self, model, ignore_index=None, lr=0.01, backbone_lr_scale=0.1, momentum=0.9, weight_decay=1e-4,
                 aux_weight=0.4, world=1, cuda_graph=False, bucket_mb=0.0, loss=None, metrics=False):
        self.model = model
        self.ignore_index, self.loss_spec = _loss_spec(loss, ignore_index)
        self._momentum, self.wd = float(momentum), float(weight_decay)
        self.aux_weight = aux_weight
        self.world = world
        self.params = [p for p in model.parameters() if p.requires_grad]
        dev = self.params[0].device
        total = sum(p.numel() for p in self.params)
        self.flat_grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_mom = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grad_views, self.mom_views = {}, []
        off = 0
        for p in self.params:
            n = p.numel()
            self.grad_views[p] = self.flat_grad[off:off + n].view(p.shape)
            self.mom_views.append(self.flat_mom[off:off + n].view(p.shape))
            off += n
        bb = set(id(p) for p in model.get_backbone_params())
        lrs = [lr * backbone_lr_scale if id(p) in bb else lr for p in self.params]
        self.base_lrs = torch.tensor(lrs, dtype=torch.float32, device=dev)
        self.lrs = self.base_lrs.clone()
        i64 = dict(dtype=torch.int64, device=dev)
        self.p_ptrs = torch.tensor([p.data_ptr() for p in self.params], **i64)
        self.g_ptrs = torch.tensor([self.grad_views[p].data_ptr() for p in self.params], **i64)
        self.m_ptrs = torch.tensor([m.data_ptr() for m in self.mom_views], **i64)
        self.sizes = torch.tensor([p.numel() for p in self.params], **i64)
        self.hyper = torch.tensor([self._momentum, self.wd], dtype=torch.float32, device=dev)  # read by the SGD kernel
        self.steps = 0
        self.wt = WeightTables(model, self.grad_views, dev)
        self.specs = self.wt.specs
        # gradient buckets (world > 1, bucket_mb > 0): contiguous ranges of the flat gradient buffer of ~bucket_mb each, in
        # parameter order; the backward produces them from the last to the first, and each bucket's all-reduce is launched on a
        # side stream as soon as its last gradient is written (SURVEY.md §8e).  The NCCL kernels then take SMs from the kernels
        # they overlap, so the default (0) is the single all-reduce after the backward
        self.bucket_mb = float(bucket_mb)
        self.buckets, self.bucket_of = [], {}
        if world > 1 and bucket_mb > 0:
            lo, acc = 0, 0
            limit = int(self.bucket_mb * (1 << 20) / 4)
            off = 0
            for p in self.params:
                self.bucket_of[p] = len(self.buckets)
                off += p.numel()
                acc += p.numel()
                if acc >= limit:
                    self.buckets.append((lo, off))
                    lo, acc = off, 0
            if acc > 0:
                self.buckets.append((lo, off))
            self.sub_unpack = self.wt.unpack_subtables(self.bucket_of)
            self.side = torch.cuda.Stream()
        # CUDA graph of the whole step (forward, loss, backward, all-reduce, SGD): ~1 200 kernel launches per step are
        # replayed by the driver instead of being re-issued from Python.  Dropout seeds and SyncBN epochs come from a
        # device-side step counter, so every replay is a fresh step.
        self.cuda_graph = cuda_graph
        self._graph = None
        self._static = None
        self._eval_graphs = {}  # (x shape, target shape) -> (static x, static target, loss, graph) of evaluate()
        self.num_classes = model.num_classes
        self.seg_counters = torch.zeros(2 + 3 * self.num_classes, dtype=torch.int64, device=dev) if metrics else None

    @property
    def momentum(self):
        return self._momentum

    @momentum.setter
    def momentum(self, value):
        """OneCycle moves the momentum every iteration: kept in device memory so graph replays see the new value."""
        if float(value) != self._momentum:
            self._momentum = float(value)
            self.hyper[0:1].fill_(self._momentum)

    def set_lr_scale(self, scale):
        """Poly / OneCycle schedules multiply the base rates (utils/lr_scheduler.py); host scalar, one tiny op."""
        torch.mul(self.base_lrs, float(scale), out=self.lrs)

    def step(self, x, target):
        if not self.cuda_graph:
            return self._step_impl(x, target)
        if self._graph is None or self._static[0].shape != x.shape or self._static[1].shape != target.shape:
            self._capture(x, target)
        self._static[0].copy_(x, non_blocking=True)
        self._static[1].copy_(target, non_blocking=True)
        self._graph.replay()
        self.steps += 1
        self._invalidate_param_caches()
        return self._static[2]

    def release_graph(self):
        """Drop the captured graphs (the step's and evaluate()'s).  Required before
        torch.distributed.destroy_process_group() when world > 1: NCCL keeps a communicator alive (and its destruction
        blocks) while a graph that captured its kernels exists."""
        torch.cuda.synchronize()
        self._graph = None
        self._static = None
        self._eval_graphs = {}
        torch.cuda.synchronize()

    def reset_metrics(self):
        """Zero the metric counters (Trainer._reset_metrics, trainer.py:173-178): one device op, no synchronisation."""
        self._require_metrics()
        self.seg_counters.zero_()

    def seg_metrics(self):
        """Trainer._get_seg_metrics (trainer.py:186-194) of everything counted since the last reset_metrics():
        {"Pixel_Accuracy", "Mean_IoU", "Class_IoU"}.  One small device-to-host copy; at world > 1 the counters are summed
        over the ranks here (one all-reduce), which gives the metrics of the batch nn.DataParallel gathers."""
        self._require_metrics()
        v = self.seg_counters
        if self.world > 1:
            v = v.clone()
            dist.all_reduce(v)
        return _metrics.seg_metrics(v.cpu().numpy(), self.num_classes)

    def _require_metrics(self):
        if self.seg_counters is None:
            raise RuntimeError("FusedTrainStep counts metrics only when constructed with metrics=True")

    def evaluate(self, x, target):
        """The per-batch work of Trainer._valid_epoch (trainer.py:125-132): an eval-mode forward of the main head
        (BatchNorm running statistics, no dropout, no SyncBN exchange), the fused upsample + loss forward with the step's
        loss (the global-batch mean under data parallel, as in training) and, with metrics=True, the counters.  Returns
        the loss as a device scalar; with cuda_graph=True it lives in a static buffer that the next evaluate() of the same
        shape overwrites.  Changes no parameter, momentum, BatchNorm buffer, dropout step counter or model.training."""
        if not self.cuda_graph:
            return self._evaluate_impl(x, target)
        key = (tuple(x.shape), tuple(target.shape))
        entry = self._eval_graphs.get(key)
        if entry is None:
            if len(self._eval_graphs) >= self.EVAL_GRAPHS_MAX:  # every graph owns a memory pool the size of the forward's
                return self._evaluate_impl(x, target)
            entry = self._eval_graphs[key] = self._capture_eval(x, target)
        xs, ys, loss, g = entry
        xs.copy_(x, non_blocking=True)
        ys.copy_(target, non_blocking=True)
        g.replay()
        return loss

    def _capture_eval(self, x, target):
        xs, ys = x.clone(), target.clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        # one eager pass outside the capture (lazy one-time initialisation, allocator pools); its counts are rolled back
        with torch.cuda.stream(side):
            saved = None if self.seg_counters is None else self.seg_counters.clone()
            self._evaluate_impl(xs, ys)
            if saved is not None:
                self.seg_counters.copy_(saved)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        if self.world > 1:  # every rank has finished its eager exchange before anyone starts capturing
            dist.barrier()
        with torch.cuda.graph(g, capture_error_mode="thread_local" if self.world > 1 else "global"):
            loss = self._evaluate_impl(xs, ys)
        return xs, ys, loss, g

    def _evaluate_impl(self, x, target):
        m = self.model
        self.wt.pack()
        tape = m._new_tape(False, False)  # eval mode: running statistics, no dropout, no step-counter increment
        tape.packed_override = self.wt.packed_bufs
        was = m.training
        m.training = False  # PSPNet builds its aux head only in training mode (pspnet.py:91); only the main head is scored
        try:
            head = m._forward_heads(tape, x.contiguous().float())[0]
        finally:
            m.training = was
        loss, _, _ = self._loss_fwd(head, target, self.seg_counters)
        return loss

    def _loss_fwd(self, head, target, counters):
        """(loss, fp64 accum, class weights) of one head.  Mean over the valid pixels of the GLOBAL batch, as
        nn.DataParallel's gathered logits give the reference (trainer.py:60-66): the (loss sum, denominator) pair is
        all-reduced (16 bytes); a 'sum' is the global sum."""
        rf = (lambda acc: dist.all_reduce(acc)) if self.world > 1 else None
        spec = self.loss_spec
        cw = spec.weight_on(head.act.t.device, head.classes)
        loss, accum = head.loss_fwd(target, self.ignore_index, cw, spec.gamma, spec.mean, reduce_fn=rf, counters=counters)
        return loss, accum, cw

    def _invalidate_param_caches(self):
        """The SGD kernel updates parameters in place without bumping autograd version counters: drop the per-parameter
        packed-weight caches the autograd/plugin path keeps, so a later model(x) call repacks the updated weights."""
        for s in self.specs:
            s._version = None

    def _capture(self, x, target):
        xs, ys = x.clone(), target.clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        # warm-up outside the capture (lazy one-time initialisation, allocator pools): two real steps whose effect on
        # the training state (parameters, momentum, BN running statistics) is rolled back afterwards
        state = [p.data for p in self.params] + [self.flat_mom] + [b for b in self.model.buffers()]
        if self.seg_counters is not None:
            state.append(self.seg_counters)
        with torch.cuda.stream(side):
            saved = [t.clone() for t in state]
            for _ in range(2):
                self._step_impl(xs, ys)
            for t, sv in zip(state, saved):
                t.copy_(sv)
            del saved
        self.steps -= 2
        cur.wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        if self.world > 1:  # every rank must have finished its eager warm-up exchanges before anyone starts capturing
            dist.barrier()
        # NCCL's all-reduce is captured with the rest (its watchdog thread polls events: relaxed capture mode)
        with torch.cuda.graph(g, capture_error_mode="thread_local" if self.world > 1 else "global"):
            loss = self._step_impl(xs, ys)
        self.steps -= 1  # the capture pass itself executed nothing
        self._graph, self._static = g, (xs, ys, loss)

    def _backward_bucketed(self, tape):
        """tape.backward() with the gradient exchange overlapped: after the closure that completes a bucket, the bucket's
        packed weight gradients are unpacked (one batched launch) and its slice of the flat buffer is all-reduced on the side
        stream while the main stream carries on with the backward.  Captured as-is by the CUDA graph of the step."""
        last = {}  # bucket -> smallest closure index writing into it (the backward runs indices downwards)
        for i, ps in tape.back_params.items():
            for p in ps:
                b = self.bucket_of.get(p)
                if b is not None and (b not in last or i < last[b]):
                    last[b] = i
        fire = {}
        for b, i in last.items():
            fire.setdefault(i, []).append(b)
        cur = torch.cuda.current_stream()
        done = set()

        def launch(b):
            done.add(b)
            tab = self.sub_unpack.get(b)
            if tab is not None:
                lib.call("seg_unpack_wgrads_batched", tab[0].data_ptr(), tab[1], tab[2], 0.0)
            ev = torch.cuda.Event()
            ev.record(cur)
            lo, hi = self.buckets[b]
            with torch.cuda.stream(self.side):
                self.side.wait_event(ev)
                dist.all_reduce(self.flat_grad[lo:hi])

        def after(i):
            for b in sorted(fire.get(i, ()), reverse=True):
                launch(b)

        tape.backward(after=after)
        for b in range(len(self.buckets) - 1, -1, -1):  # buckets no closure wrote into (frozen parameters): zeros, still exchanged
            if b not in done:
                launch(b)
        cur.wait_stream(self.side)

    def _step_impl(self, x, target):
        m = self.model
        self.flat_grad.zero_()
        self.wt.zero_wgrads()
        self.wt.pack()
        tape = m._new_tape(True, True)
        tape.grads = dict(self.grad_views)  # pre-bound views: every parameter gradient lands in the flat buffer
        tape.packed_override, tape.dw_buffers = self.wt.packed_bufs, self.wt.dw_bufs
        heads = m._forward_heads(tape, x.contiguous().float())
        total = None
        spec = self.loss_spec
        for i, head in enumerate(heads):
            # the main head only is counted (trainer.py:62); the gradient is scaled by world because the exchanged
            # gradients are averaged over ranks below
            loss, accum, cw = self._loss_fwd(head, target, self.seg_counters if i == 0 else None)
            w = 1.0 if i == 0 else self.aux_weight
            wg = w * self.world
            g = None if wg == 1.0 else torch.full((1,), wg, dtype=torch.float32, device=head.act.t.device)
            head.loss_bwd(target, self.ignore_index, accum, cw, spec.gamma, spec.mean, gscale=g)
            total = loss if total is None else total + w * loss
        m._finish(tape)
        if self.world > 1 and self.buckets:
            self._backward_bucketed(tape)
        else:
            tape.backward()
            self.wt.unpack()
            if self.world > 1:
                dist.all_reduce(self.flat_grad)
        lib.call("seg_sgd_step_dev", self.p_ptrs.data_ptr(), self.g_ptrs.data_ptr(), self.m_ptrs.data_ptr(), self.sizes.data_ptr(),
                 self.lrs.data_ptr(), len(self.params), self.hyper.data_ptr(), 0, 1.0 / self.world)
        # (momentum buffers start at zero, so "first step: buf = d" of torch.optim.SGD is the general formula)
        self._invalidate_param_caches()
        self.steps += 1
        return total
