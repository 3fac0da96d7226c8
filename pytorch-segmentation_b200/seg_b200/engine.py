"""Forward/backward engine: a tape of hand-written-kernel ops over NHWC bf16 activations.

The reference runs the hot path through torch.autograd over ATen ops (trainer.py:56,70).  Here the model's forward
is a straight-line sequence of C-ABI kernel calls recorded on a `Tape`; `Tape.backward()` replays the recorded
closures in reverse (dgrad / wgrad / BN-backward / resize-backward kernels).  torch is used for device memory only.

Conventions
  * `Act` = an activation: `.t` NHWC bf16 tensor (possibly a channel slice of a concat buffer), `.grad` its
    gradient buffer (allocated on first write; later writers accumulate with beta = 1).
  * BatchNorm (training) = statistics fused into the producing conv's epilogue -> `bn_finalize` -> one fused
    apply(+residual +ReLU +dropout) pass.  Backward = one reduce pass + one apply pass.
  * concatenation never copies: producers write into channel slices of one buffer (`Tape.concat`).
"""
import torch

from . import ops
from .lib import IMPL_AUTO, IMPL_TC

BN_EPS = 1e-5
BN_MOM = 0.1
FUSED_BWD_MAX_BYTES = 24 << 20  # BN backward: one cooperative launch up to this activation size (bf16 bytes), two above
ACT_DTYPE = torch.bfloat16  # storage type of activations / activation gradients (the kernels are bf16-only;
                            # tests/test_engine_cpu_emulated.py flips this to fp32 together with the ATen emulation)


class Act:
    __slots__ = ("t", "grad", "needs_grad", "_written")

    def __init__(self, t, needs_grad=True):
        self.t = t
        self.grad = None
        self.needs_grad = needs_grad
        self._written = False

    @property
    def shape(self):
        return self.t.shape

    def grad_target(self):
        """(buffer, beta): beta = 0 for the first writer of this gradient, 1 afterwards."""
        if self.grad is None:
            self.grad = torch.empty(self.t.shape, dtype=ACT_DTYPE, device=self.t.device)
        if not self._written:
            self._written = True
            return self.grad, 0.0
        return self.grad, 1.0


class ConvSpec:
    """Static description of one nn.Conv2d (or nn.ConvTranspose2d) holder + its packed bf16 weight cache.

    A ConvTranspose2d(Cin -> Cout, k, s, p) weight [Cin, Cout, k, k] is read as the OIHW weight of the Conv2d(Cout -> Cin, k,
    s, p) whose data gradient the transposed conv is (`transposed`; K = Cin, C = Cout): packing, the batched pack / unpack
    tables and the packed weight gradient [k*k][Cin][Cout] are those of that conv, unchanged."""

    def __init__(self, name, module, explicit_im2col=False):
        self.name = name
        self.m = module
        w = module.weight
        self.K, self.C, self.R, self.S = w.shape
        self.transposed = bool(getattr(module, "transposed", False))
        if self.transposed and (module.groups != 1 or tuple(module.dilation) != (1, 1) or tuple(module.output_padding) != (0, 0)
                                or module.bias is not None or self.R != self.S or module.stride[0] != module.stride[1]
                                or module.padding[0] != module.padding[1] or self.C % 8 != 0):
            raise NotImplementedError(f"{name}: the engine's ConvTranspose2d is square, groups 1, dilation 1, output_padding 0, "
                                      f"no bias, with a multiple of 8 output channels (got {module!r})")
        assert module.stride[0] == module.stride[1] and module.padding[0] == module.padding[1]
        assert module.dilation[0] == module.dilation[1] and module.groups == 1
        self.explicit = explicit_im2col or (self.C % 8 != 0)
        self.kpad = (self.R * self.S * self.C + 7) // 8 * 8 if self.explicit else None
        self._packed = None
        self._version = None
        self.always_repack = False  # set while a CUDA graph of the train step is captured / replayed

    @property
    def stride(self):
        return self.m.stride[0]

    @property
    def pad(self):
        return self.m.padding[0]

    @property
    def dil(self):
        return self.m.dilation[0]

    def packed_shape(self):
        return (1, self.K, self.kpad) if self.explicit else (self.R * self.S, self.K, self.C)

    def packed(self):
        w = self.m.weight
        key = (w._version, w.data_ptr())
        if self._packed is None or self._version != key or self.always_repack:
            if self.explicit:
                # column order (r, s, c): OIHW -> O,(H,W,I) as a 1x1 weight over Kpad "channels"
                w2 = w.detach().permute(0, 2, 3, 1).reshape(self.K, self.R * self.S * self.C, 1, 1).contiguous()
                self._packed = ops.pack_weight(w2, cpad=self.kpad)
            else:
                self._packed = ops.pack_weight(w.detach())
            self._version = key
        return self._packed


class DwSpec:
    """Depthwise 3x3 conv holder (nn.Conv2d with groups == channels) + packed fp32 [9][C] weight cache."""

    def __init__(self, name, module):
        self.name, self.m = name, module
        assert module.groups == module.in_channels == module.out_channels and module.kernel_size == (3, 3)
        self.C = module.in_channels
        self._packed, self._version = None, None
        self.always_repack = False

    stride = property(lambda self: self.m.stride[0])
    pad = property(lambda self: self.m.padding[0])
    dil = property(lambda self: self.m.dilation[0])

    def packed(self):
        w = self.m.weight
        key = (w._version, w.data_ptr())
        if self._packed is None or self._version != key or self.always_repack:
            self._packed = ops.dw_pack_weight(w.detach())
            self._version = key
        return self._packed


class Tape:
    def __init__(self, training, record=None, grads=None, impl=IMPL_AUTO, dropout=True, seed=0, sync=None, clamp_eps=False,
                 step_ctr=None, arena_floats=0, owner=None):
        self.training = training                                  # module.training semantics (batch stats, dropout)
        self.record = training if record is None else record      # record backward closures
        self.back = []
        self.back_params = {}  # index into self.back -> parameters whose gradient that closure writes (bucketed all-reduce)
        self.grads = grads if grads is not None else {}  # Parameter -> fp32 grad tensor (param layout)
        self.touched = set()  # parameters whose gradient this tape's backward wrote (pre-bound `grads` hide that)
        self.impl = impl
        self.dropout = dropout
        self.seed = seed
        self.sync = sync  # object with .allreduce_(fp32 vector) and .world ; None = local BN
        self.step_ctr = step_ctr  # device int64 step counter mixed into dropout seeds / SyncBN epochs (graph-replay safe)
        # FusedTrainStep hands in persistent buffers: bf16 packed weights (one batched pack launch per step) and fp32
        # packed weight-gradient accumulators (one batched unpack launch per step).  Empty for the autograd/plugin path.
        self.packed_override = {}
        self.dw_buffers = {}
        self.clamp_eps = clamp_eps
        self._drop_ctr = 0
        self._pushed = set()  # statistics vectors whose producing conv already pushed them to the SyncBN peers
        self.bn_modules = []
        # zero-initialised fp32 arena: BN-statistics accumulators and reduction slots of the whole step come out of ONE
        # zero fill instead of one fill per layer (arena_floats = what the previous step used; grows in 1M-float chunks)
        self.owner = owner  # the model: remembers how much arena a step needs
        self._arena_hint = int(arena_floats)
        self._arena = None
        self._arena_off = 0
        self.arena_used = 0

    # ------------------------------------------------------------------ helpers
    def sync_active(self):
        """SyncBN exchange on: more than one rank, or a loopback group forced on for the single-GPU protocol test."""
        s = self.sync
        return s is not None and (s.world > 1 or getattr(s, "force", False))

    def sync_fused(self):
        return self.sync_active() and getattr(self.sync, "fused", False)

    def zalloc(self, n, device):
        """n zeroed floats (128-byte aligned) from the step's arena."""
        n_al = (int(n) + 31) // 32 * 32
        if self._arena is None or self._arena_off + n_al > self._arena.numel() or self._arena.device != device:
            size = max(self._arena_hint if self._arena is None else 0, n_al, 1 << 20)
            self._arena = torch.zeros(size, dtype=torch.float32, device=device)
            self._arena_off = 0
        v = self._arena[self._arena_off:self._arena_off + int(n)]
        self._arena_off += n_al
        self.arena_used += n_al
        return v

    def zalloc64(self, n, device):
        """n zeroed fp64 words from the step's arena (the arena hands out 128-byte aligned float ranges)."""
        return self.zalloc(2 * int(n), device).view(torch.float64)

    def _param_grad(self, p, value_fn):
        """Write (or accumulate into) the fp32 gradient of parameter p.  value_fn(out, beta) fills it."""
        if not p.requires_grad:
            return
        self.touched.add(p)
        if p in self.grads:
            value_fn(self.grads[p], 1.0)
        else:
            g = torch.empty(p.shape, dtype=torch.float32, device=p.device)
            value_fn(g, 0.0)
            self.grads[p] = g

    def _push_back(self, fn, params=()):
        if params:
            self.back_params[len(self.back)] = tuple(p for p in params if p is not None)
        self.back.append(fn)

    def _unary_back(self, x, ya, fn, sole=None):
        """Record the backward of an op whose one input is x and whose output is ya (nothing when not recording), in one of
        two forms.  Accumulating (sole None): fn(dy, gx, beta) writes (beta = 0) or adds (beta = 1) x's gradient into
        x.grad_target().  Sole writer (sole = the op's name): x must have no other consumer; fn(dy) returns x's whole
        gradient, and later writers accumulate into it."""
        if not self.record:
            return

        def bwd():
            if ya.grad is None or not x.needs_grad:
                return
            if sole is None:
                gx, beta = x.grad_target()
                fn(ya.grad, gx, beta)
            else:
                assert x.grad is None, f"{sole} input must have a single consumer"
                x.grad = fn(ya.grad)
                x._written = True
            ya.grad = None
        self.back.append(bwd)

    def _drop_seed(self, drop_p):
        """(drop_p, seed) of a dropout: none outside training or with the engine's dropout off; each dropout that draws takes
        the next seed of the tape's sequence (the kernels mix in the device step counter)."""
        if not (self.training and self.dropout):
            drop_p = 0.0
        if not drop_p > 0.0:
            return drop_p, 0
        self._drop_ctr += 1
        return drop_p, (self.seed * 1000003 + self._drop_ctr * 7919) & 0x7FFFFFFFFFFFFFFF

    def _bias_grad(self, bias, dy):
        """Bias gradient = column sums of dY (fp64 accumulation); a channel count off the 8-lane pitch is read at its pitch."""
        if bias is None or not bias.requires_grad:
            return
        C, cpad = dy.shape[-1], ops.ld(dy)
        wide = dy if C % 8 == 0 else dy.as_strided(dy.shape[:-1] + (cpad,), dy.stride(), dy.storage_offset())
        s = ops.bn_stats(wide)[:C].float()
        self._param_grad(bias, lambda g, beta: g.add_(s) if beta else g.copy_(s))

    def _weight_grad(self, spec, a, b, geo, impl):
        """spec's weight gradient, conv2d_wgrad(a, b, *geo): into the trainer's persistent packed-gradient buffer (unpacked
        once per step, batched) when it has one, else unpacked into the parameter's fp32 gradient."""
        w = spec.m.weight
        if not w.requires_grad:
            return
        if spec in self.dw_buffers:
            ops.conv2d_wgrad(a, b, *geo, out=self.dw_buffers[spec], impl=impl)
            self.touched.add(w)
            return
        dwp = ops.conv2d_wgrad(a, b, *geo, impl=impl)
        if spec.explicit:
            def fill(g, beta):
                # packed [1][K][Kpad] -> [K][R,S,C] -> OIHW
                full = dwp[0, :, : spec.R * spec.S * spec.C].reshape(spec.K, spec.R, spec.S, spec.C).permute(0, 3, 1, 2)
                if beta:
                    g.add_(full)
                else:
                    g.copy_(full)
        else:
            def fill(g, beta):
                ops.unpack_wgrad(dwp, tuple(w.shape), beta=beta, out=g)
        self._param_grad(w, fill)

    def backward(self, after=None):
        """Replay the recorded closures in reverse.  after(i): called when closure i (and everything recorded after it) has
        run — the fused train step uses it to launch a gradient bucket's all-reduce as soon as the bucket is complete."""
        for i in range(len(self.back) - 1, -1, -1):
            self.back[i]()
            if after is not None:
                after(i)
        if self.owner is not None and self.arena_used:
            self.owner._arena_floats = self.arena_used
        self.back = []

    # ------------------------------------------------------------------ conv
    def conv(self, x, spec, out=None, out_dtype=None, want_stats=False, use_bias=True, stats_out=None):
        """x: Act (NHWC bf16) — or, for an explicit-im2col conv, a raw NCHW fp32 tensor (the network input).  use_bias=False
        leaves the module's bias out of the epilogue and its gradient (a consumer applies it: `score_upsample`).
        stats_out: zeroed fp64 [2K] record (a slice of a dense block's statistics table) the epilogue's statistics go to."""
        wp = self.packed_override.get(spec)
        if wp is None:
            wp = spec.packed()
        bias = spec.m.bias if use_bias else None
        stats = None
        if out_dtype is None:
            out_dtype = ACT_DTYPE
        want = want_stats and self.training
        sync = tk = None
        if want:
            # fp64 accumulators: the conv epilogue adds its column sums
            stats = self.zalloc64(2 * spec.K, wp.device) if stats_out is None else stats_out
            if self.sync_fused():  # SyncBN: the last CTA pushes the totals to the peers (no exchange launch)
                sync, tk = self.sync, self.zalloc(1, wp.device)
        if spec.explicit:
            nchw = not isinstance(x, Act)
            if not nchw and self.record and x.needs_grad and (spec.R, spec.S, spec.stride, spec.pad) != (1, 1, 1, 0):
                raise NotImplementedError(f"{spec.name}: data gradient of an im2col conv is built for 1x1 convs only")
            src = x if nchw else x.t
            col = ops.im2col(src, spec.R, spec.S, spec.stride, spec.pad, spec.dil, spec.kpad, nchw_f32=nchw)
            y = ops.conv2d_fwd(col, wp, spec.K, 1, 1, out=out, out_dtype=out_dtype, bias=bias.detach() if bias is not None else None,
                               stats=stats, impl=self.impl, sync=sync, sync_ticket=tk)
            xin, geo = col, (1, 1, 1, 0, 1)
        else:
            y = ops.conv2d_fwd(x.t, wp, spec.K, spec.R, spec.S, spec.stride, spec.pad, spec.dil, out=out, out_dtype=out_dtype,
                               bias=bias.detach() if bias is not None else None, stats=stats, impl=self.impl, sync=sync, sync_ticket=tk)
            xin, geo = x.t, (spec.R, spec.S, spec.stride, spec.pad, spec.dil)
        ya = Act(y)
        if sync is not None:
            self._pushed.add(stats.data_ptr())
        elif want and stats_out is not None:
            self.exchange_record(stats)
        if self.record:
            def bwd():
                dy = ya.grad
                if dy is None:
                    return
                self._weight_grad(spec, dy, xin, geo, self.impl)
                self._bias_grad(bias, dy)
                if (not spec.explicit) and isinstance(x, Act) and x.needs_grad:
                    gx, beta = x.grad_target()
                    ops.conv2d_dgrad(dy, wp, tuple(x.t.shape), *geo, out=gx, beta=beta, impl=self.impl)
                elif isinstance(x, Act) and x.needs_grad:
                    # 1x1 im2col conv (C % 8 != 0, e.g. DUC_out.conv over the class scores): the columns are the input padded
                    # to Kpad channels, so the dgrad over the columns is the data gradient; its pad lanes are zero because the
                    # packed weight's are
                    assert x.grad is None, "the input of an im2col conv must have a single consumer"
                    x.grad = ops.conv2d_dgrad(dy, wp, tuple(xin.shape), 1, 1, 1, 0, 1, impl=self.impl)[..., : spec.C]
                    x._written = True
                ya.grad = None
            self._push_back(bwd, (spec.m.weight, bias))
        return ya, stats

    def conv_transpose(self, x, spec, out=None):
        """nn.ConvTranspose2d (spec.transposed) of x [N,h,w,Cin] -> [N,(h-1)s-2p+k,(w-1)s-2p+k,Cout]; `out` may be a concat slice.
        forward = the dgrad of the Conv2d(Cout -> Cin) (its stride-s parity classes write the strided sub-grids of the
        output), data gradient = that conv's fprop over dY, weight gradient = its wgrad with the operands swapped.  The
        wgmma kernels run these shapes; AUTO therefore asks for them (IMPL_TC), so an unsupported call raises instead of
        silently taking the CUDA-core path."""
        assert spec.transposed
        wp = self.packed_override.get(spec)
        if wp is None:
            wp = spec.packed()
        impl = IMPL_TC if self.impl == IMPL_AUTO else self.impl
        k, s, p = spec.R, spec.stride, spec.pad
        N, h, w, _ = x.t.shape
        y_shape = (N, (h - 1) * s - 2 * p + k, (w - 1) * s - 2 * p + k, spec.C)
        y = ops.conv2d_dgrad(x.t, wp, y_shape, k, k, s, p, 1, out=out, impl=impl)
        ya = Act(y)
        if self.record:
            def bwd():
                dy = ya.grad
                if dy is None:
                    return
                self._weight_grad(spec, x.t, dy, (k, k, s, p, 1), impl)
                if x.needs_grad:
                    gx, beta = x.grad_target()
                    ops.conv2d_fwd(dy, wp, spec.K, k, k, s, p, 1, out=gx, beta=beta, impl=impl)
                ya.grad = None
            self._push_back(bwd, (spec.m.weight,))
        return ya

    def dwconv(self, x, spec, want_stats=False):
        """Depthwise 3x3 (SeparableConv2d.conv1).  Returns (raw output Act, BN statistics or None)."""
        w9 = spec.packed()
        stats = self.zalloc64(2 * spec.C, w9.device) if (want_stats and self.training) else None
        sync = self.sync if (stats is not None and self.sync_fused()) else None
        y = ops.dwconv_fwd(x.t, w9, spec.stride, spec.pad, spec.dil, stats=stats, sync=sync,
                           sync_ticket=self.zalloc(1, w9.device) if sync is not None else None)
        if sync is not None:
            self._pushed.add(stats.data_ptr())
        ya = Act(y)
        if self.record:
            def bwd():
                dy = ya.grad
                if dy is None:
                    return
                if spec.m.weight.requires_grad:
                    g9 = ops.dwconv_bwd_weight(dy, x.t, spec.stride, spec.pad, spec.dil)
                    self._param_grad(spec.m.weight, lambda g, beta: ops.dw_unpack_wgrad(g9, g, beta))
                if x.needs_grad:
                    gx, beta = x.grad_target()
                    ops.dwconv_bwd_data(dy, w9, tuple(x.t.shape), spec.stride, spec.pad, spec.dil, out=gx, beta=beta)
                ya.grad = None
            self._push_back(bwd, (spec.m.weight,))
        return ya, stats

    def relu(self, x):
        y = ops.relu_fwd(x.t)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.relu_bwd(dy, y, gx, beta))
        return ya

    # ------------------------------------------------------------------ dense-block statistics table
    def exchange_record(self, stats):
        """A statistics record a producer wrote into a dense block's table: with an exchange object that has no in-kernel
        protocol (the gloo stand-in), sum it over the ranks here, once — its consumers (every later layer's norm1) never
        exchange a prefix."""
        if self.sync_active() and stats.data_ptr() not in self._pushed:
            self.sync.allreduce_(stats)
            self._pushed.add(stats.data_ptr())

    def record_stats(self, x, stats):
        """bn_stats of x (a slice of a dense block's buffer) into its zeroed table record, exchanged once."""
        if not self.training:
            return
        sync0 = self.sync if self.sync_fused() else None
        ops.bn_stats(x.t, stats=stats, sync=sync0)
        if sync0 is not None:
            self._pushed.add(stats.data_ptr())
        self.exchange_record(stats)

    # ------------------------------------------------------------------ batch norm (+ residual, ReLU, dropout)
    def bn_act(self, y, bn, stats=None, relu=True, res=None, out=None, drop_p=0.0, drop_channelwise=False, table=None):
        """y: Act holding the raw conv output.  Returns the activated Act.  drop_channelwise: nn.Dropout2d semantics (one
        draw per image and channel, models/pspnet.py:22,68) instead of nn.Dropout's per-element draws.
        table = (stats table, c0, growth): pre-activation BN over a dense block's channel prefix y (`prefix`): the batch
        statistics come from the block's table (records exchanged by their producers), and the backward ADDS the data
        gradient into y's gradient (a view of the block's) as its first writer's beta dictates."""
        drop_hw = y.t.shape[1] * y.t.shape[2] if drop_channelwise else 0
        C = y.t.shape[-1]
        count_local = ops.rows(y.t)
        use_batch_stats = self.training and bn.training
        drop_p, seed = self._drop_seed(drop_p)
        # conv -> BN(batch statistics) -> ReLU with nothing in between: the ReLU mask can be recomputed from the conv output
        # with the forward's own coefficients instead of being read (the one-launch backward of the small maps does so)
        remask = bool(use_batch_stats and relu and res is None and drop_p == 0.0)
        mask_kw = {}
        table_kw, acc_kw = {}, {}
        if table is not None:
            if use_batch_stats:
                stats, table_kw = table[0], {"table": (table[1], table[2])}
            else:
                stats = None
        if use_batch_stats:
            if stats is None:
                sync0 = self.sync if self.sync_fused() else None
                stats = ops.bn_stats(y.t, sync=sync0)
                if sync0 is not None:
                    self._pushed.add(stats.data_ptr())
            count = count_local
            if self.sync_active():
                # a producer called with sync= has already exchanged: `stats` holds the world's totals
                if stats.data_ptr() not in self._pushed and table is None:
                    # exchange object without the in-kernel protocol (the gloo stand-in of the CPU tests): sums over ranks
                    self.sync.allreduce_(stats)
                count = count_local * self.sync.world
            # the ReLU mask of the backward passes as bits, written by the forward apply: 1/16 of the bytes of re-reading
            # the activation, and on the large maps faster than recomputing it too (the reduce's recomputing variant
            # needs 74 registers: 3 blocks/SM instead of 4).  Not written where the one-launch backward recomputes it
            # (remask on a small map).  A kernel layer without the bit mask (the ATen stand-in of the host-logic tests)
            # reads the activation.
            if relu and hasattr(ops, "relu_mask") and not (remask and count_local * C * 2 <= FUSED_BWD_MAX_BYTES):
                mask_kw = {"mask": ops.relu_mask(y.t)}
            # finalize (coefficients, saved mean / 1/std, running statistics) happens inside the apply kernel
            a, save = ops.bn_apply_train(y.t, stats, count, bn.weight.detach(), bn.bias.detach(), bn.eps,
                                         bn.momentum if bn.momentum is not None else BN_MOM,
                                         1 if (self.clamp_eps and self.sync is not None and self.sync.world > 1) else 0,
                                         bn.running_mean, bn.running_var, res=res.t if res is not None else None, out=out,
                                         relu=relu, drop_p=drop_p, seed=seed, step_ctr=self.step_ctr if drop_p > 0.0 else None,
                                         drop_hw=drop_hw, **mask_kw, **table_kw)
            self.bn_modules.append(bn)
        else:
            ss, save = ops.bn_eval_scale_shift(bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var, bn.eps,
                                               want_save=True)
            count = count_local
            a = ops.bn_apply(y.t, ss, res=res.t if res is not None else None, out=out, relu=relu, drop_p=drop_p, seed=seed,
                             step_ctr=self.step_ctr if drop_p > 0.0 else None, drop_hw=drop_hw)
        aa = Act(a)
        if self.record:
            def bwd():
                da = aa.grad
                if da is None:
                    return
                want_pg = bn.weight.requires_grad
                acc_pg = want_pg and (bn.weight in self.grads)
                if want_pg:
                    self.touched.update((bn.weight, bn.bias))
                if want_pg and not acc_pg:
                    self.grads[bn.weight] = torch.empty(C, dtype=torch.float32, device=a.device)
                    self.grads[bn.bias] = torch.empty(C, dtype=torch.float32, device=a.device)
                a_mask = None if remask else a  # the bit mask in mask_kw takes precedence
                acc_kw = {}
                if table is not None:
                    dy, beta_dx = y.grad_target()
                    if beta_dx:
                        acc_kw = {"beta_dx": beta_dx}
                else:
                    dy = torch.empty(y.t.shape, dtype=ACT_DTYPE, device=a.device)
                dres, beta_res = (None, 0.0)
                if res is not None and res.needs_grad:
                    dres, beta_res = res.grad_target()
                sync = self.sync if (use_batch_stats and self.sync_active()) else None
                dg = self.grads[bn.weight] if want_pg else None
                db = self.grads[bn.bias] if want_pg else None
                if sync is not None and not getattr(sync, "fused", False):
                    # exchange object without the in-kernel protocol (the gloo stand-in of the CPU tests)
                    sums = ops.bn_bwd_reduce(da, a, y.t, save, relu=relu, drop_p=drop_p, dgamma=dg, dbeta=db, accumulate=acc_pg,
                                             acc=self.zalloc64(ops.bn_bwd_reduce_acc_words(C), a.device), **mask_kw)
                    gsums = sums.clone()
                    sync.allreduce_(gsums)
                    ops.bn_bwd_apply(da, a_mask, y.t, save, bn.weight.detach(), gsums, count, relu=relu, drop_p=drop_p, dx=dy,
                                     dres=dres, beta_res=beta_res, beta=bn.bias.detach(), **mask_kw, **acc_kw)
                elif count_local * C * 2 <= FUSED_BWD_MAX_BYTES:
                    # small maps (the operands stay in L2 between the phases): reduce -> grid barrier -> fixed-order cross-block
                    # sum (-> SyncBN exchange) -> apply in ONE cooperative launch.  Frozen BN (freeze_bn): dx = gamma*inv_std*dz,
                    # the sums only feed the parameter gradients.  Its one ticket (seg_bn_bwd_fused_workspace) is the
                    # grid-barrier counter
                    ops.bn_bwd_fused(da, a_mask, y.t, save, bn.weight.detach(), count, relu=relu, drop_p=drop_p, dgamma=dg, dbeta=db,
                                     accumulate=acc_pg, dx=dy, dres=dres, beta_res=beta_res, beta=bn.bias.detach(),
                                     zero_sums=not use_batch_stats, tickets=self.zalloc(1, a.device), sync=sync, **mask_kw, **acc_kw)
                else:
                    # large maps stream from HBM in both passes anyway: two launches at full occupancy; under SyncBN the
                    # reduction's last block exchanges the sums, so the apply pass gets the world's
                    sums = ops.bn_bwd_reduce(da, a, y.t, save, relu=relu, drop_p=drop_p, dgamma=dg, dbeta=db, accumulate=acc_pg,
                                             acc=self.zalloc64(ops.bn_bwd_reduce_acc_words(C), a.device), sync=sync, **mask_kw)
                    gsums = sums if use_batch_stats else torch.zeros_like(sums)
                    ops.bn_bwd_apply(da, a_mask, y.t, save, bn.weight.detach(), gsums, count, relu=relu, drop_p=drop_p, dx=dy,
                                     dres=dres, beta_res=beta_res, beta=bn.bias.detach(), **mask_kw, **acc_kw)
                y.grad = dy
                aa.grad = None
            self._push_back(bwd, (bn.weight, bn.bias))
        return aa

    # ------------------------------------------------------------------ pooling / resize / concat
    def maxpool(self, x):
        """nn.MaxPool2d(3, 2, 1) of a ResNet stem.  x must be the pool's only consumer."""
        y, idx = ops.maxpool3x3s2_fwd(x.t)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy: ops.maxpool3x3s2_bwd(dy, idx, tuple(x.t.shape)), sole="maxpool")
        return ya

    def maxpool2x2(self, x):
        """nn.MaxPool2d(2, 2, return_indices=True) (segnet.py:30).  Returns (pooled Act, record): the record holds the
        codes and the pre-pool shape, for `maxunpool2x2`.  x must be the pool's only consumer (as in SegNet)."""
        y, code = ops.maxpool2x2_fwd(x.t)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy: ops.maxpool2x2_bwd(dy, code, tuple(x.t.shape)), sole="maxpool2x2")
        return ya, (code, tuple(x.t.shape))

    def maxunpool2x2(self, x, record):
        """nn.MaxUnpool2d(2, 2) of x to the pre-pool size of the max-pool that wrote `record` (segnet.py:106-118).  x must
        be the unpool's only consumer (as in SegNet)."""
        code, shape = record
        y = ops.maxunpool2x2_fwd(x.t, code, shape[1:3])
        ya = Act(y)
        self._unary_back(x, ya, lambda dy: ops.maxunpool2x2_bwd(dy, code), sole="maxunpool2x2")
        return ya

    def relu_maxpool_ceil(self, x):
        """F.relu then nn.MaxPool2d(2, 2, ceil_mode=True) of the raw conv output x (FCN8's VGG stages, fcn.py:20-22), one
        kernel each way; the backward writes every element of x's gradient.  x must be the pool's only consumer."""
        y, code = ops.relu_maxpool2x2_ceil_fwd(x.t)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy: ops.relu_maxpool2x2_ceil_bwd(dy, code, tuple(x.t.shape)), sole="relu_maxpool_ceil")
        return ya

    def relu_dropout(self, x, drop_p):
        """F.relu then nn.Dropout(drop_p) (FCN8's conv6 / conv7, fcn.py:49-51); a plain ReLU outside training or with the
        engine's dropout off.  Masks: bn_act's seed sequence and the device step counter."""
        drop_p, seed = self._drop_seed(drop_p)
        y = ops.relu_dropout_fwd(x.t, drop_p, seed, self.step_ctr if drop_p > 0.0 else None)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.relu_dropout_bwd(dy, y, drop_p, gx, beta))
        return ya

    def score_upsample(self, x, up, window, skip=None, skip_off=(0, 0), alpha=0.0, bias=None, out_dtype=None):
        """Window (y0, x0, Ho, Wo) of the frozen nn.ConvTranspose2d `up` (C -> C, k = 2s, stride s, no padding) over the class
        map x, plus alpha * skip[window at skip_off] + bias when a skip is given — FCN8's `adj_poolN(alpha * poolN)[crop] +
        up(...)` (fcn.py:86-97) with the adj conv run by `conv(..., use_bias=False)` into `skip`.  One launch each way; the
        backward writes x's gradient, the skip's (alpha * dY in the window, 0 elsewhere) and adds the bias gradient (column
        sums of dY).  x and skip must have no other consumer.  `up` gets no gradient: a trainable weight raises."""
        if up.weight.requires_grad:
            raise NotImplementedError("score_upsample: the engine computes no gradient for the upsampling weight; keep it frozen "
                                      "(requires_grad=False), as models/fcn.py does")
        k = up.kernel_size[0]
        wf = ops.score_pack(up.weight, bwd=False)
        wb = ops.score_pack(up.weight, bwd=True) if self.record else None
        y = ops.score_upsample_fwd(x.t, wf, k, window, skip=skip.t if skip is not None else None, skip_off=skip_off, alpha=alpha,
                                   bias=bias.detach() if bias is not None else None, out_dtype=out_dtype or ACT_DTYPE)
        ya = Act(y)
        if self.record:
            def bwd():
                dy = ya.grad
                if dy is None:
                    return
                self._bias_grad(bias, dy)
                if skip is not None and skip.needs_grad:
                    assert skip.grad is None, "score_upsample skip must have a single consumer"
                    skip.grad = ops.score_skip_bwd(dy, tuple(skip.t.shape), skip_off, alpha)
                    skip._written = True
                if x.needs_grad:
                    assert x.grad is None, "score_upsample input must have a single consumer"
                    x.grad = ops.score_upsample_bwd(dy, wb, tuple(x.t.shape), k, window)
                    x._written = True
                ya.grad = None
            self._push_back(bwd, (bias,))
        return ya

    def avgpool2x2(self, x, out=None):
        """nn.AvgPool2d(2, 2), floor mode (DenseNet's transition1), into `out` (a channel slice of the next block's buffer)."""
        y = ops.avgpool2x2_fwd(x.t, out=out)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.avgpool2x2_bwd(dy, tuple(x.t.shape), dx=gx, beta=beta))
        return ya

    def avgpool(self, x, bins):
        y = ops.adaptive_avgpool_fwd(x.t, bins)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.adaptive_avgpool_bwd(dy, tuple(x.t.shape), bins, dx=gx, beta=beta))
        return ya

    def bilinear(self, x, Ho, Wo, align_corners, out=None):
        y = ops.bilinear_fwd(x.t, Ho, Wo, align_corners, out=out)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.bilinear_bwd(dy, x.t.shape[1], x.t.shape[2], align_corners, dx=gx,
                                                                      beta=beta))
        return ya

    def pixel_shuffle(self, x, r, out=None, crop=None):
        """nn.PixelShuffle(r) of x [N,H,W,r*r*C], cropped to crop = (Ho, Wo) (default r*H x r*W); `out`: a concat slice."""
        N, H, W, _ = x.t.shape
        Ho, Wo = crop if crop is not None else (H * r, W * r)
        y = ops.pixel_shuffle_fwd(x.t, r, Ho, Wo, out=out)
        ya = Act(y)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.pixel_shuffle_bwd(dy, r, H, W, dx=gx, beta=beta))
        return ya

    def up_add(self, x, y):
        """up_and_add of the reference's FPN (models/upernet.py:89-90): bilinear(x -> size of y, align_corners=True) + y."""
        Hy, Wy = y.t.shape[1], y.t.shape[2]
        u = ops.bilinear_fwd(x.t, Hy, Wy, True)
        ops.axpby(y.t, u, 1.0)  # u += y
        ua = Act(u)
        if self.record:
            def bwd():
                g = ua.grad
                if g is None:
                    return
                if y.needs_grad:
                    gy, beta = y.grad_target()
                    ops.axpby(g, gy, beta)
                if x.needs_grad:
                    gx, beta = x.grad_target()
                    ops.bilinear_bwd(g, x.t.shape[1], x.t.shape[2], True, dx=gx, beta=beta)
                ua.grad = None
            self.back.append(bwd)
        return ua

    def copy_into(self, x, out):
        """Copy an activation into a concat slice (used when the producer's tensor is also consumed elsewhere)."""
        ops.axpby(x.t, out, 0.0)
        ya = Act(out)
        self._unary_back(x, ya, lambda dy, gx, beta: ops.axpby(dy, gx, beta))
        return ya

    def concat(self, N, H, W, channels, device):
        """Allocate one NHWC buffer; returns (whole Act, [slice tensors]).  Producers pass a slice as `out=`; call
        `bind_slices` with the producer Acts so their gradients alias slices of the whole gradient."""
        total = sum(channels)
        buf = torch.empty((N, H, W, total), dtype=ACT_DTYPE, device=device)
        whole = Act(buf)
        slices, off = [], 0
        for c in channels:
            slices.append(buf[..., off:off + c])
            off += c
        return whole, slices

    def pitched(self, N, H, W, C, device):
        """Activation buffer [N,H,W,C] with channel pitch ceil8(C), for class maps (C = the class count): the kernels that
        produce and consume them touch the C class lanes only."""
        return torch.empty((N, H, W, (C + 7) // 8 * 8), dtype=ACT_DTYPE, device=device)[..., :C]

    def bind_slices(self, whole, acts):
        """After the producers ran: make each producer Act's gradient a view of the concat gradient buffer."""
        if not self.record:
            return
        g = whole.grad  # pre-allocated by `dense_buffer`
        if g is None:
            g = torch.empty(whole.t.shape, dtype=ACT_DTYPE, device=whole.t.device)
        whole.grad = g
        off = 0
        for a in acts:
            c = a.t.shape[-1]
            a.grad = g[..., off:off + c]
            off += c
        whole._written = False  # the consumer's dgrad overwrites (beta = 0) the pre-allocated buffer

    def dense_buffer(self, N, H, W, C, device):
        """A dense block's NHWC buffer: its producers write channel slices in place and its layers read prefixes (`prefix`).
        Its gradient buffer exists from the start, so the prefix views can be bound before the backward runs; the block's
        downstream consumer writes it first (beta = 0), every later writer adds."""
        whole = Act(torch.empty((N, H, W, C), dtype=ACT_DTYPE, device=device))
        if self.record:
            whole.grad = torch.empty((N, H, W, C), dtype=ACT_DTYPE, device=device)
        return whole

    def prefix(self, whole, c0, c1=None, act=None):
        """Channels [c0, c1) of a `dense_buffer` as an Act whose gradient is the matching view of the block's gradient,
        written before any consumer of the view runs its backward (so every writer accumulates).  act: the Act of the
        producer that wrote those channels in place, bound instead of a new one."""
        c1 = whole.t.shape[-1] if c1 is None else c1
        a = Act(whole.t[..., c0:c1]) if act is None else act
        if whole.grad is not None:
            a.grad = whole.grad[..., c0:c1]
            a._written = True
        return a

    def shared_slice(self, act):
        """`act` was produced into a concat slice (and bound by `bind_slices`) and has consumers of its own besides the
        concat's (a skip connection taken from the residual stream).  Call right after `bind_slices`: in the backward this
        runs once the concat's consumer has written the slice (beta = 0), so act's own consumers then ADD to it."""
        if self.record:
            def bwd():
                act._written = True
            self.back.append(bwd)


# ---------------------------------------------------------------------- output heads
# A head owns how a model's last tape activation becomes the full-resolution NCHW fp32 logits `model(x)` returns, and the
# fused loss that reads those logits in place (FusedTrainStep).  Both write the gradient of that activation.
class BilinearHead:
    """Low-resolution NHWC fp32 logits, bilinearly upsampled to (H, W) (deeplabv3_plus.py:361, pspnet.py:86, upernet.py:143)."""

    def __init__(self, act, align_corners, H, W):
        self.act, self.align_corners, self.H, self.W = act, align_corners, H, W

    @property
    def classes(self):
        return self.act.t.shape[-1]

    def logits(self):
        return ops.bilinear_logits_fwd(self.act.t, self.H, self.W, self.align_corners)

    def logits_bwd(self, dout):
        C, t = self.classes, self.act.t
        self.act.grad = ops.bilinear_logits_bwd(dout, t.shape[1], t.shape[2], self.align_corners, (C + 7) // 8 * 8)[..., :C]

    def loss_fwd(self, target, ignore_index, weight, gamma, mean, reduce_fn=None, counters=None):
        loss, accum, _ = ops.upsample_loss_fwd(self.act.t, target, self.align_corners, ignore_index, weight, gamma, mean,
                                               reduce_fn=reduce_fn, counters=counters)
        return loss, accum

    def loss_bwd(self, target, ignore_index, accum, weight, gamma, mean, gscale=None):
        C = self.classes
        dx, _ = ops.upsample_loss_bwd(self.act.t, target, self.align_corners, ignore_index, accum, (C + 7) // 8 * 8, weight, gamma,
                                      mean, gscale=gscale)
        self.act.grad = dx[..., :C]


class ShuffleHead:
    """NHWC bf16 map [N,h,w,r*r*C] whose nn.PixelShuffle(r) is the output [N,C,r*h,r*w] (DeepLab_DUC_HDC, duc_hdc.py:233)."""

    def __init__(self, act, r):
        self.act, self.r = act, r

    @property
    def classes(self):
        return self.act.t.shape[-1] // (self.r * self.r)

    def _ld(self):
        return (self.act.t.shape[-1] + 7) // 8 * 8

    def logits(self):
        return ops.pixel_shuffle_logits_fwd(self.act.t, self.r)

    def logits_bwd(self, dout):
        self.act.grad = ops.pixel_shuffle_logits_bwd(dout, self.r, self._ld())[..., : self.act.t.shape[-1]]

    def loss_fwd(self, target, ignore_index, weight, gamma, mean, reduce_fn=None, counters=None):
        return ops.shuffle_loss_fwd(self.act.t, self.r, target, ignore_index, weight, gamma, mean, reduce_fn=reduce_fn,
                                    counters=counters)

    def loss_bwd(self, target, ignore_index, accum, weight, gamma, mean, gscale=None):
        dx = ops.shuffle_loss_bwd(self.act.t, self.r, target, ignore_index, accum, self._ld(), weight, gamma, mean, gscale=gscale)
        self.act.grad = dx[..., : self.act.t.shape[-1]]


class FullResHead:
    """NHWC fp32 logits [N,H,W,C] (a pitch is allowed) already at the output resolution (UNetResnet's conv7, unet.py:204)."""

    def __init__(self, act):
        self.act = act

    @property
    def classes(self):
        return self.act.t.shape[-1]

    def _ld(self):
        return (self.classes + 7) // 8 * 8

    def logits(self):
        return ops.nhwc_to_nchw_f32(self.act.t)

    def logits_bwd(self, dout):
        # the NCHW fp32 -> NHWC bf16 transpose with zero pad lanes is the pixel shuffle's at r = 1
        self.act.grad = ops.pixel_shuffle_logits_bwd(dout, 1, self._ld())[..., : self.classes]

    def loss_fwd(self, target, ignore_index, weight, gamma, mean, reduce_fn=None, counters=None):
        return ops.nhwc_loss_fwd(self.act.t, target, ignore_index, weight, gamma, mean, reduce_fn=reduce_fn, counters=counters)

    def loss_bwd(self, target, ignore_index, accum, weight, gamma, mean, gscale=None):
        dx = ops.nhwc_loss_bwd(self.act.t, target, ignore_index, accum, self._ld(), weight, gamma, mean, gscale=gscale)
        self.act.grad = dx[..., : self.classes]
