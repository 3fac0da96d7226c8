"""Tensor-level wrappers over the C ABI (one Python function per ``seg_*`` entry point).

Activations are NHWC ``torch.bfloat16`` tensors; a tensor may be a channel slice ``buf[..., a:b]`` of a wider
buffer (that is how concatenation is expressed — no copy).  These wrappers only compute shapes / pitches and pass
raw pointers; all arithmetic happens in the sm_90a kernels.
"""
import ctypes

import torch

from . import lib
from .lib import DT_BF16, DT_F32, IMPL_AUTO, IMPL_SIMT, IMPL_TC, ConvDesc, call, make_conv_desc, ptr

_IMPL_OVERRIDE = None
PROFILE = None  # set to a list to record (kind, algorithmic flops, start event, end event) for every conv launch


def _meta(d):
    if lib.TRACE is None:
        return None
    return (d.N, d.H, d.W, d.C, d.K, d.R, d.stride, d.dil, 2.0 * d.N * d.P * d.Q * d.K * d.C * d.R * d.S)


def _meta_rows(M, C, passes, flag=0):
    """Trace metadata of a streaming kernel: (rows, channels, flag) and its algorithmic bytes (bf16 passes over M x C)."""
    if lib.TRACE is None:
        return None
    return (int(M), int(C), int(flag), 0, 0, 0, 0, 0, 2.0 * M * C * passes)


def _prof(kind, d):
    """Context helper: CUDA events on the launching stream around one conv launch (bench.py's roofline leg)."""
    if PROFILE is None:
        return None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    flops = 2.0 * d.N * d.P * d.Q * d.K * d.C * d.R * d.S
    # algorithmic bytes of the launch: both bf16 activation operands once + the weights (bf16 fprop/dgrad, fp32 wgrad output)
    nbytes = 2.0 * (d.N * d.H * d.W * d.C + d.N * d.P * d.Q * d.K) + (4.0 if kind == "wgrad" else 2.0) * d.K * d.C * d.R * d.S
    PROFILE.append((kind, flops, e0, e1, nbytes))
    e0.record()
    return e1


def set_conv_impl(impl):
    """Force a conv implementation (IMPL_AUTO / IMPL_SIMT / IMPL_TC) for every conv call; None restores per-call choice."""
    global _IMPL_OVERRIDE
    _IMPL_OVERRIDE = impl


def _impl(impl):
    return _IMPL_OVERRIDE if _IMPL_OVERRIDE is not None else impl


def ld(t):
    """Channel pitch of an NHWC (or [M, C]) tensor; checks the slice is addressable as rows of `ld` elements."""
    assert t.stride(-1) == 1, "channel dim must be contiguous"
    if t.dim() == 4:
        n, h, w, c = t.shape
        pitch = t.stride(2) if w > 1 else (t.stride(1) // w if h > 1 else (t.stride(0) // (h * w) if n > 1 else c))
        assert w == 1 or t.stride(2) == pitch
        assert h == 1 or t.stride(1) == w * pitch, "rows must be dense"
        assert n == 1 or t.stride(0) == h * w * pitch, "images must be dense"
        return pitch
    return t.stride(-2) if t.shape[-2] > 1 else t.shape[-1]


def rows(t):
    m = 1
    for s in t.shape[:-1]:
        m *= s
    return m


# ---------------------------------------------------------------- conv
def pack_weight(w_oihw, cpad=None):
    K, C, R, S = w_oihw.shape
    cpad = cpad or C
    out = torch.empty((R * S, K, cpad), dtype=torch.bfloat16, device=w_oihw.device)
    call("seg_pack_weight", ptr(w_oihw), ptr(out), K, C, R, S, cpad)
    return out


def unpack_wgrad(dw_packed, shape, beta=0.0, out=None):
    K, C, R, S = shape
    cpad = dw_packed.shape[-1]
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=dw_packed.device)
        beta = 0.0
    call("seg_unpack_wgrad", ptr(dw_packed), ptr(out), K, C, R, S, cpad, float(beta))
    return out


def conv_desc_for(x, K, R, S, stride, pad, dil, ldy=None):
    N, H, W, C = x.shape
    return make_conv_desc(N, H, W, C, K, R, S, stride, pad, dil, ldx=ld(x), ldy=ldy)


_WS_CACHE = {}


def new_stats(C, device):
    """Zeroed fp64 [2C] accumulator for BatchNorm batch statistics (sum, sum of squares) — the producers ADD into it."""
    return torch.zeros(2 * C, dtype=torch.float64, device=device)


def _sync_args(sync, ticket, device):
    """(desc pointer, ticket pointer, ticket tensor kept alive) for a SyncBN producer call."""
    if sync is None:
        return None, None, None
    if ticket is None:
        ticket = torch.zeros(1, dtype=torch.float32, device=device)
    return ctypes.addressof(sync.desc), ptr(ticket), ticket


def conv2d_fwd(x, w_packed, K, R, S, stride=1, pad=0, dil=1, out=None, out_dtype=torch.bfloat16, bias=None, beta=0.0,
               stats=None, impl=IMPL_AUTO, sync=None, sync_ticket=None):
    """stats: fp64 [2K], ZERO on entry (new_stats): the per-channel sum / sum of squares of the output are added to it
    (exact fp64 accumulation: bit-reproducible).  sync: a comm.SyncBNGroup — the last CTA also pushes the totals to every
    peer; sync_ticket: one zeroed word from the caller's arena (allocated here if None)."""
    N, H, W, C = x.shape
    d = make_conv_desc(N, H, W, C, K, R, S, stride, pad, dil, ldx=ld(x))
    if out is None:
        out = torch.empty((N, d.P, d.Q, K), dtype=out_dtype, device=x.device)
    d.ldy = ld(out)
    assert stats is None or stats.dtype == torch.float64
    sp, tp, _keep = _sync_args(sync if stats is not None else None, sync_ticket, x.device)
    ev = _prof("fprop", d)
    call("seg_conv2d_fwd", ctypes.byref(d), ptr(x), ptr(w_packed), ptr(out), DT_BF16 if out.dtype == torch.bfloat16 else DT_F32,
         ptr(bias), float(beta), ptr(stats), sp, tp, _impl(impl), meta=_meta(d))
    if ev is not None:
        ev.record()
    return out


def conv2d_dgrad(dy, w_packed, x_shape, R, S, stride=1, pad=0, dil=1, out=None, beta=0.0, impl=IMPL_AUTO):
    N, H, W, C = x_shape
    K = dy.shape[-1]
    if out is None:
        out = torch.empty((N, H, W, C), dtype=torch.bfloat16, device=dy.device)
        beta = 0.0
    d = make_conv_desc(N, H, W, C, K, R, S, stride, pad, dil, ldx=ld(out), ldy=ld(dy))
    assert (d.P, d.Q) == (dy.shape[1], dy.shape[2])
    ev = _prof("dgrad", d)
    call("seg_conv2d_dgrad", ctypes.byref(d), ptr(dy), ptr(w_packed), ptr(out), float(beta), _impl(impl), meta=_meta(d))
    if ev is not None:
        ev.record()
    return out


def conv2d_wgrad(dy, x, R, S, stride=1, pad=0, dil=1, out=None, impl=IMPL_AUTO):
    """Returns / accumulates into fp32 packed grad [R*S][K][C]."""
    N, H, W, C = x.shape
    K = dy.shape[-1]
    if out is None:
        out = torch.zeros((R * S, K, C), dtype=torch.float32, device=x.device)
    d = make_conv_desc(N, H, W, C, K, R, S, stride, pad, dil, ldx=ld(x), ldy=ld(dy))
    assert (d.P, d.Q) == (dy.shape[1], dy.shape[2])
    nws = lib.load().seg_conv2d_wgrad_workspace_floats(ctypes.byref(d), _impl(impl))
    if nws < 0:
        raise RuntimeError(f"seg_conv2d_wgrad_workspace_floats failed: {lib.last_error()}")
    ws = torch.empty(nws, dtype=torch.float32, device=x.device) if nws > 0 else None
    ev = _prof("wgrad", d)
    call("seg_conv2d_wgrad", ctypes.byref(d), ptr(dy), ptr(x), ptr(out), ptr(ws), _impl(impl), meta=_meta(d))
    if ev is not None:
        ev.record()
    return out


# ---------------------------------------------------------------- depthwise 3x3
def dw_pack_weight(w_c133):
    C = w_c133.shape[0]
    w9 = torch.empty((9, C), dtype=torch.float32, device=w_c133.device)
    call("seg_dw_pack_weight", ptr(w_c133), ptr(w9), C)
    return w9


def dw_unpack_wgrad(g9, out, beta=0.0):
    call("seg_dw_unpack_wgrad", ptr(g9), ptr(out), g9.shape[1], float(beta))
    return out


def _dw_desc(x_shape, stride, pad, dil, ldx, ldy):
    N, H, W, C = x_shape
    return make_conv_desc(N, H, W, C, C, 3, 3, stride, pad, dil, ldx=ldx, ldy=ldy)


def dwconv_fwd(x, w9, stride=1, pad=1, dil=1, out=None, stats=None, sync=None, sync_ticket=None):
    N, H, W, C = x.shape
    d = _dw_desc(x.shape, stride, pad, dil, ld(x), C)
    if out is None:
        out = torch.empty((N, d.P, d.Q, C), dtype=torch.bfloat16, device=x.device)
    d.ldy = ld(out)
    assert stats is None or stats.dtype == torch.float64
    sp, tp, _keep = _sync_args(sync if stats is not None else None, sync_ticket, x.device)
    call("seg_dwconv3x3_fwd", ctypes.byref(d), ptr(x), ptr(w9), ptr(out), ptr(stats), sp, tp)
    return out


def dwconv_bwd_data(dy, w9, x_shape, stride=1, pad=1, dil=1, out=None, beta=0.0):
    if out is None:
        out = torch.empty(x_shape, dtype=torch.bfloat16, device=dy.device)
        beta = 0.0
    d = _dw_desc(x_shape, stride, pad, dil, ld(out), ld(dy))
    assert (d.P, d.Q) == (dy.shape[1], dy.shape[2])
    call("seg_dwconv3x3_bwd_data", ctypes.byref(d), ptr(dy), ptr(w9), ptr(out), float(beta))
    return out


def dwconv_bwd_weight(dy, x, stride=1, pad=1, dil=1, out=None, beta=0.0):
    C = x.shape[-1]
    if out is None:
        out = torch.empty((9, C), dtype=torch.float32, device=x.device)
        beta = 0.0
    d = _dw_desc(x.shape, stride, pad, dil, ld(x), ld(dy))
    scratch = torch.empty(int(lib.load().seg_dwconv_scratch_floats(C)) // 2 + 1, dtype=torch.float64, device=x.device)
    call("seg_dwconv3x3_bwd_weight", ctypes.byref(d), ptr(dy), ptr(x), ptr(out), float(beta), ptr(scratch))
    return out


def im2col(x, R, S, stride, pad, dil, kpad, nchw_f32):
    if nchw_f32:
        N, C, H, W = x.shape
        ldx = C
    else:
        N, H, W, C = x.shape
        ldx = ld(x)
    d = make_conv_desc(N, H, W, C, 1, R, S, stride, pad, dil, ldx=ldx, ldy=1)
    col = torch.empty((N, d.P, d.Q, kpad), dtype=torch.bfloat16, device=x.device)
    call("seg_im2col", ctypes.byref(d), ptr(x), 1 if nchw_f32 else 0, ptr(col), kpad)
    return col


# ---------------------------------------------------------------- batch norm
def bn_stats(x, stats=None, sync=None, sync_ticket=None):
    """fp64 [2C] (sum, sum of squares) over the rows of x (added to `stats`, which must be zero on entry if given)."""
    C = x.shape[-1]
    if stats is None:
        stats = new_stats(C, x.device)
    sp, tp, _keep = _sync_args(sync, sync_ticket, x.device)
    call("seg_bn_stats", ptr(x), rows(x), C, ld(x), ptr(stats), sp, tp)
    return stats


def bn_finalize(stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var):
    C = gamma.numel()
    ss = torch.empty(2 * C, dtype=torch.float32, device=stats.device)
    save = torch.empty(2 * C, dtype=torch.float32, device=stats.device)
    call("seg_bn_finalize", ptr(stats), float(count), C, ptr(gamma), ptr(beta), float(eps), float(momentum), int(clamp_eps),
         ptr(running_mean), ptr(running_var), ptr(ss), ptr(save))
    return ss, save


def bn_eval_scale_shift(gamma, beta, rm, rv, eps, want_save=False):
    C = gamma.numel()
    ss = torch.empty(2 * C, dtype=torch.float32, device=gamma.device)
    save = torch.empty(2 * C, dtype=torch.float32, device=gamma.device) if want_save else None
    call("seg_bn_eval_scale_shift", C, ptr(gamma), ptr(beta), ptr(rm), ptr(rv), float(eps), ptr(ss), ptr(save))
    return (ss, save) if want_save else ss


def bn_apply(x, scale_shift, res=None, out=None, relu=True, drop_p=0.0, seed=0, step_ctr=None, drop_hw=0):
    C = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    call("seg_bn_apply", ptr(x), ld(x), ptr(scale_shift), ptr(res), ld(res) if res is not None else 0, ptr(out), ld(out),
         rows(x), C, int(relu), float(drop_p), int(seed), ptr(step_ctr), int(drop_hw))
    return out


def counter_add(ctr, inc=1):
    call("seg_counter_add", ptr(ctr), int(inc))


MASK_PASS = 1.0 / 16  # the ReLU bit mask: 1 bit per element, in bf16 passes over M x C


def relu_mask(x):
    """Uninitialised ReLU bit-mask buffer for the activation of BN over x (bn_apply_train(mask=) fills it, the backward
    passes read it): uint8 [M][C/8], bit j of [m][g] = activation[m][8g+j] > 0; its own pitch C/8, whatever the
    activation's channel pitch."""
    return torch.empty((rows(x), x.shape[-1] // 8), dtype=torch.uint8, device=x.device)


def _check_mask(mask, x):
    if mask is not None:
        assert mask.dtype == torch.uint8 and mask.is_contiguous() and tuple(mask.shape) == (rows(x), x.shape[-1] // 8), \
            "mask: uint8 [M][C/8] from relu_mask()"


def _mask_passes(relu, out, mask):
    """bf16 passes over M x C the backward spends on the ReLU mask: the bits, the activation, or none (recomputed)."""
    if not relu:
        return 0
    return MASK_PASS if mask is not None else (1 if out is not None else 0)


def bn_bwd_reduce_acc_words(C):
    """fp64 words of the zeroed accumulator block of bn_bwd_reduce: [slots][2C] sums + one ticket word."""
    return int(lib.load().seg_bn_bwd_reduce_slots()) * 2 * C + 1


def bn_bwd_reduce(dout, out, x, save, relu=True, drop_p=0.0, dgamma=None, dbeta=None, accumulate=False, acc=None,
                  gamma=None, beta=None, sync=None, mask=None):
    """Returns sums fp32 [2C] = (sum dz, sum dz*xhat); optionally writes the parameter gradients from them.  One launch: fp64
    atomics into `acc` (exact, bit-reproducible), the last block rounds / writes.  acc: zeroed fp64 [bn_bwd_reduce_acc_words(C)]
    (accumulator copies + ticket) from the caller's arena, allocated here if None.  sync: SyncBN — the last block exchanges the sums with the
    peers and the returned sums are the world's.
    out=None (with relu, gamma, beta): the ReLU mask is recomputed from x instead of read from the stored activation.
    mask: the ReLU bit mask bn_apply_train wrote for this activation (read instead of out)."""
    C = x.shape[-1]
    M = rows(x)
    sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    nw = bn_bwd_reduce_acc_words(C)
    if acc is None:
        acc = torch.zeros(nw, dtype=torch.float64, device=x.device)
    assert acc.dtype == torch.float64 and acc.numel() >= nw
    _check_mask(mask, x)
    call("seg_bn_bwd_reduce", ptr(dout), ld(dout), ptr(out), ld(out) if out is not None else 0, ptr(mask), ptr(x), ld(x), ptr(save),
         M, C, int(relu), float(drop_p), ptr(sums), ptr(acc), acc.data_ptr() + 8 * (nw - 1), ptr(dgamma), ptr(dbeta), int(accumulate),
         ptr(gamma), ptr(beta), ctypes.addressof(sync.desc) if sync is not None else None,
         meta=_meta_rows(M, C, 2 + _mask_passes(relu, out, mask)))
    return sums


def bn_apply_train(x, stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var, res=None, out=None,
                   relu=True, drop_p=0.0, seed=0, step_ctr=None, drop_hw=0, mask=None, table=None):
    """Training-mode BN (+residual, ReLU, dropout) straight from the batch sums.  Returns (out, save[2C]).
    Under SyncBN the producer called with sync= has left the world's sums in `stats`; `count` is then the world's.
    mask (with relu): relu_mask(x) buffer, filled with the ReLU bit mask of out for the backward passes.
    table = (c0, growth): `stats` is a dense block's statistics table (records [sum, sum^2] of width c0, then growth, back to
    back in channel order) and x the block buffer's channel prefix [0, C)."""
    C = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    save = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    assert stats.dtype == torch.float64
    c0, growth = table if table is not None else (0, 0)
    if table is not None:
        assert growth > 0 and 0 < c0 <= C and (C - c0) % growth == 0, f"table {table} does not tile {C} channels"
        assert stats.is_contiguous() and stats.numel() >= 2 * C, "statistics table too short"
    _check_mask(mask, x)
    call("seg_bn_apply_train", ptr(x), ld(x), ptr(stats), float(count), ptr(gamma), ptr(beta), float(eps), float(momentum),
         int(clamp_eps), ptr(running_mean), ptr(running_var), ptr(save), ptr(res), ld(res) if res is not None else 0,
         ptr(out), ld(out), ptr(mask), rows(x), C, int(relu), float(drop_p), int(seed), ptr(step_ctr), int(drop_hw), int(c0),
         int(growth), meta=_meta_rows(rows(x), C, (3 if res is not None else 2) + (MASK_PASS if mask is not None else 0), res is not None))
    return out, save


def bn_bwd_apply(dout, out, x, save, gamma, sums, count, relu=True, drop_p=0.0, dx=None, dres=None, beta_res=0.0, beta=None,
                 mask=None, beta_dx=0.0):
    """beta_dx = 1: dx += the BN data gradient (fp32 sum, one bf16 rounding) instead of dx = it."""
    C = x.shape[-1]
    if dx is None:
        dx = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
        beta_dx = 0.0
    _check_mask(mask, x)
    call("seg_bn_bwd_apply", ptr(dout), ld(dout), ptr(out), ld(out) if out is not None else 0, ptr(mask), ptr(x), ld(x), ptr(save),
         ptr(gamma), ptr(sums), float(count), rows(x), C, int(relu), float(drop_p), ptr(dx), ld(dx), ptr(dres),
         ld(dres) if dres is not None else 0, float(beta_res), ptr(beta), float(beta_dx),
         meta=_meta_rows(rows(x), C, 2 + _mask_passes(relu, out, mask) + (2 if beta_dx else 1) + (0 if dres is None else (2 if beta_res != 0.0 else 1)), dres is not None))
    return dx


def bn_bwd_fused_workspace(M, C):
    key = ("bnf", int(M), int(C))
    v = _WS_CACHE.get(key)
    if v is None:
        r, t = ctypes.c_int64(), ctypes.c_int64()
        if lib.load().seg_bn_bwd_fused_workspace(int(M), int(C), ctypes.byref(r), ctypes.byref(t)) != 0:
            raise RuntimeError(lib.last_error())
        v = _WS_CACHE[key] = (int(r.value), int(t.value))
    return v


def bn_bwd_fused(dout, out, x, save, gamma, count_total, relu=True, drop_p=0.0, dgamma=None, dbeta=None, accumulate=False,
                 dx=None, dres=None, beta_res=0.0, beta=None, zero_sums=False, tickets=None, sync=None, mask=None, beta_dx=0.0):
    """BatchNorm backward in ONE cooperative launch (reduce -> grid barrier -> fixed-order cross-block sum [-> SyncBN exchange]
    -> apply).  Returns (dx, sums [2C]: the world's under sync).  out=None: ReLU mask recomputed from x (needs beta).  tickets:
    bn_bwd_fused_workspace(M, C)[1] zeroed words.  mask: ReLU bit mask from bn_apply_train (read instead of out).
    beta_dx = 1: dx += the BN data gradient (fp32 sum, one bf16 rounding)."""
    C = x.shape[-1]
    M = rows(x)
    if dx is None:
        dx = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
        beta_dx = 0.0
    sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    nr, nt = bn_bwd_fused_workspace(M, C)
    fr = torch.empty(max(nr, 1), dtype=torch.float32, device=x.device)
    if tickets is None:
        tickets = torch.zeros(max(nt, 1), dtype=torch.float32, device=x.device)
    _check_mask(mask, x)
    call("seg_bn_bwd_fused", ptr(dout), ld(dout), ptr(out), ld(out) if out is not None else 0, ptr(mask), ptr(x), ld(x), ptr(save), ptr(gamma),
         ptr(beta), float(count_total), M, C, int(relu), float(drop_p), ptr(sums), ptr(fr), ptr(tickets), ptr(dgamma), ptr(dbeta),
         int(accumulate), ptr(dx), ld(dx), ptr(dres), ld(dres) if dres is not None else 0, float(beta_res), int(zero_sums),
         ctypes.addressof(sync.desc) if sync is not None else None, float(beta_dx),
         meta=_meta_rows(M, C, (2 + _mask_passes(relu, out, mask)) * 2 + (2 if beta_dx else 1) + (0 if dres is None else (2 if beta_res != 0.0 else 1)), dres is not None))
    return dx, sums


def bn_param_grad(sums, dgamma, dbeta, accumulate=False):
    C = sums.numel() // 2
    call("seg_bn_param_grad", ptr(sums), C, ptr(dgamma), ptr(dbeta), int(accumulate))


# ---------------------------------------------------------------- pooling / resize
def maxpool3x3s2_fwd(x):
    N, H, W, C = x.shape
    P, Q = lib.conv_out_size(H, 3, 2, 1, 1), lib.conv_out_size(W, 3, 2, 1, 1)
    assert x.is_contiguous()
    y = torch.empty((N, P, Q, C), dtype=torch.bfloat16, device=x.device)
    idx = torch.empty((N, P, Q, C), dtype=torch.uint8, device=x.device)
    call("seg_maxpool3x3s2_fwd", ptr(x), ptr(y), ptr(idx), N, H, W, C, P, Q)
    return y, idx


def maxpool3x3s2_bwd(dy, idx, x_shape):
    N, H, W, C = x_shape
    P, Q = dy.shape[1], dy.shape[2]
    assert dy.is_contiguous()
    dx = torch.empty(x_shape, dtype=torch.bfloat16, device=dy.device)
    call("seg_maxpool3x3s2_bwd", ptr(dy), ptr(idx), ptr(dx), N, H, W, C, P, Q)
    return dx


def maxpool2x2_fwd(x):
    """nn.MaxPool2d(2, 2, return_indices=True), floor mode: (y [N,H//2,W//2,C] bf16, codes uint8 of y's shape, 2r + s)."""
    N, H, W, C = x.shape
    assert x.is_contiguous()
    y = torch.empty((N, H // 2, W // 2, C), dtype=torch.bfloat16, device=x.device)
    code = torch.empty(y.shape, dtype=torch.uint8, device=x.device)
    call("seg_maxpool2x2_fwd", ptr(x), ptr(y), ptr(code), N, H, W, C)
    return y, code


def maxpool2x2_bwd(dy, code, x_shape):
    N, H, W, C = x_shape
    assert dy.is_contiguous() and tuple(dy.shape) == (N, H // 2, W // 2, C) and code.shape == dy.shape
    dx = torch.empty(x_shape, dtype=torch.bfloat16, device=dy.device)
    call("seg_maxpool2x2_bwd", ptr(dy), ptr(code), ptr(dx), N, H, W, C)
    return dx


def maxunpool2x2_fwd(x, code, out_hw):
    """nn.MaxUnpool2d(2, 2) with output_size = out_hw, the pre-pool size whose max-pool wrote `code`."""
    N, P, Q, C = x.shape
    H, W = out_hw
    assert x.is_contiguous() and (P, Q) == (H // 2, W // 2) and code.shape == x.shape
    y = torch.empty((N, H, W, C), dtype=torch.bfloat16, device=x.device)
    call("seg_maxunpool2x2_fwd", ptr(x), ptr(code), ptr(y), N, H, W, C)
    return y


def maxunpool2x2_bwd(dy, code):
    N, H, W, C = dy.shape
    assert dy.is_contiguous() and tuple(code.shape) == (N, H // 2, W // 2, C)
    dx = torch.empty(code.shape, dtype=torch.bfloat16, device=dy.device)
    call("seg_maxunpool2x2_bwd", ptr(dy), ptr(code), ptr(dx), N, H, W, C)
    return dx


def relu_maxpool2x2_ceil_fwd(x):
    """F.relu then nn.MaxPool2d(2, 2, ceil_mode=True) of the raw conv output x: (y [N,ceil(H/2),ceil(W/2),C] bf16, codes uint8
    of y's shape: 2r + s, plus 4 where the window max is <= 0 and the gradient is dropped)."""
    N, H, W, C = x.shape
    assert x.is_contiguous()
    y = torch.empty((N, (H + 1) // 2, (W + 1) // 2, C), dtype=torch.bfloat16, device=x.device)
    code = torch.empty(y.shape, dtype=torch.uint8, device=x.device)
    call("seg_relu_maxpool2x2_ceil_fwd", ptr(x), ptr(y), ptr(code), N, H, W, C)
    return y, code


def relu_maxpool2x2_ceil_bwd(dy, code, x_shape):
    N, H, W, C = x_shape
    assert dy.is_contiguous() and tuple(dy.shape) == (N, (H + 1) // 2, (W + 1) // 2, C) and code.shape == dy.shape
    dx = torch.empty(x_shape, dtype=torch.bfloat16, device=dy.device)
    call("seg_relu_maxpool2x2_ceil_bwd", ptr(dy), ptr(code), ptr(dx), N, H, W, C)
    return dx


def avgpool2x2_fwd(x, out=None):
    """nn.AvgPool2d(2, 2) (floor mode) of x [N,H,W,C] -> [N,H//2,W//2,C]; `out` may be a channel slice of a concat buffer."""
    N, H, W, C = x.shape
    if out is None:
        out = torch.empty((N, H // 2, W // 2, C), dtype=torch.bfloat16, device=x.device)
    assert tuple(out.shape) == (N, H // 2, W // 2, C)
    call("seg_avgpool2x2_fwd", ptr(x), ld(x), ptr(out), ld(out), N, H, W, C, meta=_meta_rows(N * H * W, C, 1.25))
    return out


def avgpool2x2_bwd(dy, x_shape, dx=None, beta=0.0):
    """dx = beta * dx + the pool's data gradient over every element of dx (0 for a dropped odd row / column)."""
    N, H, W, C = x_shape
    assert tuple(dy.shape) == (N, H // 2, W // 2, C)
    if dx is None:
        dx = torch.empty(x_shape, dtype=torch.bfloat16, device=dy.device)
        beta = 0.0
    call("seg_avgpool2x2_bwd", ptr(dy), ld(dy), ptr(dx), ld(dx), N, H, W, C, float(beta),
         meta=_meta_rows(N * H * W, C, 1.25 + (1 if beta else 0)))
    return dx


def adaptive_avgpool_fwd(x, bins):
    N, H, W, C = x.shape
    y = torch.empty((N, bins, bins, C), dtype=torch.bfloat16, device=x.device)
    call("seg_adaptive_avgpool_fwd", ptr(x), ld(x), ptr(y), N, H, W, C, bins)
    return y


def adaptive_avgpool_bwd(dy, x_shape, bins, dx=None, beta=0.0):
    N, H, W, C = x_shape
    assert dy.is_contiguous()
    if dx is None:
        dx = torch.empty(x_shape, dtype=torch.bfloat16, device=dy.device)
        beta = 0.0
    call("seg_adaptive_avgpool_bwd", ptr(dy), ptr(dx), ld(dx), N, H, W, C, bins, float(beta))
    return dx


def bilinear_fwd(x, Ho, Wo, align_corners, out=None):
    N, Hi, Wi, C = x.shape
    if out is None:
        out = torch.empty((N, Ho, Wo, C), dtype=torch.bfloat16, device=x.device)
    call("seg_bilinear_fwd", ptr(x), ld(x), ptr(out), ld(out), N, Hi, Wi, Ho, Wo, C, int(align_corners))
    return out


def bilinear_bwd(dy, Hi, Wi, align_corners, dx=None, beta=0.0):
    N, Ho, Wo, C = dy.shape
    if dx is None:
        dx = torch.empty((N, Hi, Wi, C), dtype=torch.bfloat16, device=dy.device)
        beta = 0.0
    call("seg_bilinear_bwd", ptr(dy), ld(dy), ptr(dx), ld(dx), N, Hi, Wi, Ho, Wo, C, int(align_corners), float(beta))
    return dx


def bilinear_logits_fwd(x_nhwc_f32, Ho, Wo, align_corners):
    N, Hi, Wi, C = x_nhwc_f32.shape
    assert x_nhwc_f32.is_contiguous() and x_nhwc_f32.dtype == torch.float32
    y = torch.empty((N, C, Ho, Wo), dtype=torch.float32, device=x_nhwc_f32.device)
    call("seg_bilinear_logits_fwd", ptr(x_nhwc_f32), ptr(y), N, Hi, Wi, Ho, Wo, C, int(align_corners))
    return y


def bilinear_logits_bwd(dy_nchw, Hi, Wi, align_corners, ldx):
    N, C, Ho, Wo = dy_nchw.shape
    assert dy_nchw.is_contiguous() and dy_nchw.dtype == torch.float32
    dx = torch.empty((N, Hi, Wi, ldx), dtype=torch.bfloat16, device=dy_nchw.device)
    call("seg_bilinear_logits_bwd", ptr(dy_nchw), ptr(dx), ldx, N, Hi, Wi, Ho, Wo, C, int(align_corners))
    return dx


def pixel_shuffle_fwd(x, r, Ho, Wo, out=None):
    """nn.PixelShuffle(r) on NHWC bf16 [N,H,W,r*r*C], cropped to [N,Ho,Wo,C] (Ho <= r*H, Wo <= r*W); `out` may be a channel slice."""
    N, H, W, Cr = x.shape
    C = Cr // (r * r)
    assert C * r * r == Cr and x.dtype == torch.bfloat16
    if out is None:
        out = torch.empty((N, Ho, Wo, C), dtype=torch.bfloat16, device=x.device)
    assert tuple(out.shape) == (N, Ho, Wo, C)
    call("seg_pixel_shuffle_fwd", ptr(x), ld(x), ptr(out), ld(out), N, H, W, C, r, Ho, Wo)
    return out


def pixel_shuffle_bwd(dy, r, H, W, dx=None, beta=0.0):
    """dx [N,H,W,r*r*C] = beta*dx + the inverse permutation of dy [N,Ho,Wo,C]; positions the crop dropped get zero."""
    N, Ho, Wo, C = dy.shape
    if dx is None:
        dx = torch.empty((N, H, W, C * r * r), dtype=torch.bfloat16, device=dy.device)
        beta = 0.0
    assert tuple(dx.shape) == (N, H, W, C * r * r)
    call("seg_pixel_shuffle_bwd", ptr(dy), ld(dy), ptr(dx), ld(dx), N, H, W, C, r, Ho, Wo, float(beta))
    return dx


def pixel_shuffle_logits_fwd(x, r):
    """NHWC bf16 [N,h,w,r*r*C] -> the NCHW fp32 [N,C,r*h,r*w] logits of F.pixel_shuffle."""
    N, h, w, Cr = x.shape
    C = Cr // (r * r)
    assert C * r * r == Cr and x.dtype == torch.bfloat16
    y = torch.empty((N, C, h * r, w * r), dtype=torch.float32, device=x.device)
    call("seg_pixel_shuffle_logits_fwd", ptr(x), ld(x), ptr(y), N, h, w, C, r)
    return y


def pixel_shuffle_logits_bwd(dy_nchw, r, ldx):
    """NCHW fp32 grad [N,C,r*h,r*w] -> NHWC bf16 [N,h,w,ldx] (channels r*r*C.. zero)."""
    N, C, Ho, Wo = dy_nchw.shape
    assert dy_nchw.is_contiguous() and dy_nchw.dtype == torch.float32 and Ho % r == 0 and Wo % r == 0
    dx = torch.empty((N, Ho // r, Wo // r, ldx), dtype=torch.bfloat16, device=dy_nchw.device)
    call("seg_pixel_shuffle_logits_bwd", ptr(dy_nchw), ptr(dx), ldx, N, Ho // r, Wo // r, C, r)
    return dx


# ---------------------------------------------------------------- loss
def _loss_kind(weight, gamma, mean):
    """SEG_LOSS_* of a per-pixel loss: focal when gamma is given; else unweighted cross-entropy for a mean without class
    weights; else class-weighted cross-entropy (weight None = all ones)."""
    if gamma is not None:
        return lib.LOSS_FOCAL
    return lib.LOSS_CE if weight is None and mean else lib.LOSS_WCE


def loss_nchw_fwd(logits, target, ignore_index, weight=None, gamma=None, mean=True, reduce_fn=None):
    """Cross-entropy, class-weighted CE or focal loss (gamma >= 0) on NCHW fp32 logits; weight: fp32 [C] device tensor or
    None.  Returns (loss, accum); accum = fp64 (per-pixel loss sum, denominator).  reduce_fn(accum): optional in-place
    cross-rank sum of accum before the loss is formed.  mean=False: the loss is the (globally reduced) sum."""
    N, C, H, W = logits.shape
    assert logits.is_contiguous() and logits.dtype == torch.float32 and target.dtype == torch.int64 and target.is_contiguous()
    assert weight is None or (weight.dtype == torch.float32 and weight.numel() == C and weight.is_contiguous())
    accum = torch.zeros(2, dtype=torch.float64, device=logits.device)
    call("seg_loss_nchw_fwd", ptr(logits), ptr(target), N, C, H, W, int(ignore_index), ptr(weight), _loss_kind(weight, gamma, mean),
         float(gamma or 0.0), ptr(accum))
    if reduce_fn is not None:
        reduce_fn(accum)
    loss = torch.empty((), dtype=torch.float32, device=logits.device)
    call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
    return loss, accum


def loss_nchw_bwd(logits, target, ignore_index, accum, weight=None, gamma=None, mean=True, gscale=None):
    N, C, H, W = logits.shape
    dl = torch.empty_like(logits)
    call("seg_loss_nchw_bwd", ptr(logits), ptr(target), N, C, H, W, int(ignore_index), ptr(weight), _loss_kind(weight, gamma, mean),
         float(gamma or 0.0), int(mean), ptr(accum), ptr(gscale), ptr(dl))
    return dl


def dice_nchw_fwd(logits, target, smooth=1.0):
    N, C, H, W = logits.shape
    assert logits.is_contiguous() and logits.dtype == torch.float32 and target.dtype == torch.int64 and target.is_contiguous()
    accum = torch.zeros(2, dtype=torch.float64, device=logits.device)
    loss = torch.empty((), dtype=torch.float32, device=logits.device)
    call("seg_dice_nchw_fwd", ptr(logits), ptr(target), N, C, H, W, float(smooth), ptr(accum), ptr(loss))
    return loss, accum


def dice_nchw_bwd(logits, target, accum, smooth=1.0, gscale=None, out=None, beta=0.0):
    N, C, H, W = logits.shape
    if out is None:
        out = torch.empty_like(logits)
        beta = 0.0
    call("seg_dice_nchw_bwd", ptr(logits), ptr(target), N, C, H, W, ptr(accum), float(smooth), ptr(gscale), ptr(out), float(beta))
    return out


def lovasz_softmax_nchw(logits, target, ignore_index):
    """Returns (loss scalar tensor, dlogits NCHW fp32).  One host sync to size the key buffers."""
    N, C, H, W = logits.shape
    assert logits.is_contiguous() and logits.dtype == torch.float32 and target.dtype == torch.int64 and target.is_contiguous()
    dev = logits.device
    counts = torch.empty(C + 1, dtype=torch.int32, device=dev)
    call("seg_lovasz_count", ptr(target), N * H * W, C, int(ignore_index), ptr(counts))
    ch = counts.cpu()
    P, n_present = int(ch[C]), int((ch[:C] > 0).sum())
    nkeys = max(P * n_present, 1)
    keys0 = torch.empty(nkeys, dtype=torch.int64, device=dev)
    keys1 = torch.empty(nkeys, dtype=torch.int64, device=dev)
    ws = torch.empty(int(lib.load().seg_lovasz_workspace_bytes(P, n_present, C)), dtype=torch.uint8, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    dl = torch.empty_like(logits)
    call("seg_lovasz_softmax_nchw", ptr(logits), ptr(target), N, C, H, W, int(ignore_index), ptr(counts), P, n_present,
         ptr(keys0), ptr(keys1), ptr(ws), ptr(loss), ptr(dl))
    return loss, dl


def eval_metrics_nchw(logits, target, num_class):
    """int64 device vector [2 + 3K]: correct, labeled, area_inter[K], area_pred[K], area_lab[K]."""
    N, C, H, W = logits.shape
    assert logits.is_contiguous() and logits.dtype == torch.float32 and target.dtype == torch.int64 and target.is_contiguous()
    out = torch.empty(2 + 3 * num_class, dtype=torch.int64, device=logits.device)
    call("seg_eval_metrics_nchw", ptr(logits), ptr(target), N, C, H, W, int(num_class), ptr(out))
    return out


def _check_counters(counters, C):
    assert counters.dtype == torch.int64 and counters.is_contiguous() and counters.numel() == 2 + 3 * C


def upsample_loss_fwd(logits_lo, target, align_corners, ignore_index, weight=None, gamma=None, mean=True, want_argmax=False,
                      reduce_fn=None, counters=None):
    """loss_nchw_fwd fused with the bilinear upsample of the low-res NHWC fp32 logits; returns (loss, accum, argmax map or
    None).  counters: None, or an int64 device vector [2 + 3C] that the same launch ADDS the batch's eval_metrics counters
    to (the layout of eval_metrics_nchw with num_class = C)."""
    N, Hi, Wi, C = logits_lo.shape
    _, Ho, Wo = target.shape
    assert logits_lo.is_contiguous() and logits_lo.dtype == torch.float32 and target.is_contiguous()
    assert weight is None or (weight.dtype == torch.float32 and weight.numel() == C and weight.is_contiguous())
    if counters is not None:
        _check_counters(counters, C)
    accum = torch.zeros(2, dtype=torch.float64, device=logits_lo.device)
    am = torch.empty((N, Ho, Wo), dtype=torch.int32, device=logits_lo.device) if want_argmax else None
    call("seg_upsample_loss_fwd", ptr(logits_lo), ptr(target), N, Hi, Wi, Ho, Wo, C, int(align_corners), int(ignore_index),
         ptr(weight), _loss_kind(weight, gamma, mean), float(gamma or 0.0), ptr(accum), ptr(am), ptr(counters))
    if reduce_fn is not None:
        reduce_fn(accum)
    loss = torch.empty((), dtype=torch.float32, device=logits_lo.device)
    call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
    return loss, accum, am


def upsample_loss_bwd(logits_lo, target, align_corners, ignore_index, accum, ldx, weight=None, gamma=None, mean=True,
                      gscale=None):
    N, Hi, Wi, C = logits_lo.shape
    _, Ho, Wo = target.shape
    dlo = torch.empty((N, Hi, Wi, C), dtype=torch.float32, device=logits_lo.device)
    fixed = torch.empty((N, Hi, Wi, C), dtype=torch.int64, device=logits_lo.device)
    dx = torch.empty((N, Hi, Wi, ldx), dtype=torch.bfloat16, device=logits_lo.device)
    call("seg_upsample_loss_bwd", ptr(logits_lo), ptr(target), N, Hi, Wi, Ho, Wo, C, int(align_corners), int(ignore_index),
         ptr(weight), _loss_kind(weight, gamma, mean), float(gamma or 0.0), int(mean), ptr(accum), ptr(gscale), ptr(dlo),
         ptr(fixed), ptr(dx), ldx)
    return dx, dlo


def _shuffle_loss_shapes(lo, r, target):
    N, h, w, Cr = lo.shape
    C = Cr // (r * r)
    assert C * r * r == Cr and lo.dtype == torch.bfloat16 and target.dtype == torch.int64 and target.is_contiguous()
    if tuple(target.shape) != (N, h * r, w * r):
        raise ValueError(f"target size {tuple(target.shape[1:])} differs from the model output size {(h * r, w * r)}")
    return N, h, w, C


def shuffle_loss_fwd(logits_lo, r, target, ignore_index, weight=None, gamma=None, mean=True, reduce_fn=None, counters=None):
    """loss_nchw_fwd on the F.pixel_shuffle(r) view of the NHWC bf16 map [N,h,w,r*r*C], read in place; returns (loss, accum).
    counters: as for upsample_loss_fwd."""
    N, h, w, C = _shuffle_loss_shapes(logits_lo, r, target)
    assert weight is None or (weight.dtype == torch.float32 and weight.numel() == C and weight.is_contiguous())
    if counters is not None:
        _check_counters(counters, C)
    accum = torch.zeros(2, dtype=torch.float64, device=logits_lo.device)
    call("seg_shuffle_loss_fwd", ptr(logits_lo), ld(logits_lo), ptr(target), N, h, w, C, r, int(ignore_index), ptr(weight),
         _loss_kind(weight, gamma, mean), float(gamma or 0.0), ptr(accum), ptr(counters))
    if reduce_fn is not None:
        reduce_fn(accum)
    loss = torch.empty((), dtype=torch.float32, device=logits_lo.device)
    call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
    return loss, accum


def shuffle_loss_bwd(logits_lo, r, target, ignore_index, accum, ldx, weight=None, gamma=None, mean=True, gscale=None):
    """Gradient of shuffle_loss_fwd's loss w.r.t. the low-res map: bf16 [N,h,w,ldx] (channels r*r*C.. zero)."""
    N, h, w, C = _shuffle_loss_shapes(logits_lo, r, target)
    dx = torch.empty((N, h, w, ldx), dtype=torch.bfloat16, device=logits_lo.device)
    call("seg_shuffle_loss_bwd", ptr(logits_lo), ld(logits_lo), ptr(target), N, h, w, C, r, int(ignore_index), ptr(weight),
         _loss_kind(weight, gamma, mean), float(gamma or 0.0), int(mean), ptr(accum), ptr(gscale), ptr(dx), ldx)
    return dx


def _nhwc_loss_shapes(logits, target):
    N, H, W, C = logits.shape
    assert logits.dtype == torch.float32 and target.dtype == torch.int64 and target.is_contiguous()
    if tuple(target.shape) != (N, H, W):
        raise ValueError(f"target size {tuple(target.shape[1:])} differs from the model output size {(H, W)}")
    return N, H, W, C


def nhwc_loss_fwd(logits, target, ignore_index, weight=None, gamma=None, mean=True, reduce_fn=None, counters=None):
    """loss_nchw_fwd on full-resolution NHWC fp32 logits [N,H,W,C] (a pitch is allowed), read in place; returns (loss, accum).
    counters: as for upsample_loss_fwd."""
    N, H, W, C = _nhwc_loss_shapes(logits, target)
    assert weight is None or (weight.dtype == torch.float32 and weight.numel() == C and weight.is_contiguous())
    if counters is not None:
        _check_counters(counters, C)
    accum = torch.zeros(2, dtype=torch.float64, device=logits.device)
    call("seg_nhwc_loss_fwd", ptr(logits), ld(logits), ptr(target), N, H, W, C, int(ignore_index), ptr(weight),
         _loss_kind(weight, gamma, mean), float(gamma or 0.0), ptr(accum), ptr(counters))
    if reduce_fn is not None:
        reduce_fn(accum)
    loss = torch.empty((), dtype=torch.float32, device=logits.device)
    call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
    return loss, accum


def nhwc_loss_bwd(logits, target, ignore_index, accum, ldx, weight=None, gamma=None, mean=True, gscale=None):
    """Gradient of nhwc_loss_fwd's loss w.r.t. the logits: bf16 [N,H,W,ldx] (channels C.. zero)."""
    N, H, W, C = _nhwc_loss_shapes(logits, target)
    dx = torch.empty((N, H, W, ldx), dtype=torch.bfloat16, device=logits.device)
    call("seg_nhwc_loss_bwd", ptr(logits), ld(logits), ptr(target), N, H, W, C, int(ignore_index), ptr(weight),
         _loss_kind(weight, gamma, mean), float(gamma or 0.0), int(mean), ptr(accum), ptr(gscale), ptr(dx), ldx)
    return dx


# ---------------------------------------------------------------- misc
def nhwc_to_nchw_f32(x):
    N, H, W, C = x.shape
    y = torch.empty((N, C, H, W), dtype=torch.float32, device=x.device)
    call("seg_nhwc_to_nchw_f32", ptr(x), ld(x), DT_BF16 if x.dtype == torch.bfloat16 else DT_F32, ptr(y), N, H, W, C)
    return y


def relu_fwd(x):
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    call("seg_relu_fwd", ptr(x), ld(x), ptr(y), ld(y), rows(x), x.shape[-1])
    return y


def relu_bwd(dy, y, dx, beta):
    call("seg_relu_bwd", ptr(dy), ld(dy), ptr(y), ld(y), ptr(dx), ld(dx), rows(y), y.shape[-1], float(beta))
    return dx


def relu_dropout_fwd(x, drop_p, seed=0, step_ctr=None):
    """relu(x) then nn.Dropout(drop_p) in training (drop_p = 0: F.relu); masks from bn_apply's hash stream."""
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    call("seg_relu_dropout_fwd", ptr(x), ld(x), ptr(y), ld(y), rows(x), x.shape[-1], float(drop_p), int(seed), ptr(step_ctr))
    return y


def relu_dropout_bwd(dy, y, drop_p, dx, beta):
    call("seg_relu_dropout_bwd", ptr(dy), ld(dy), ptr(y), ld(y), ptr(dx), ld(dx), rows(y), y.shape[-1], float(drop_p), float(beta))
    return dx


# ---------------------------------------------------------------- class-map transposed conv (FCN8's score upsamplers)
def score_pack(w, bwd):
    """ConvTranspose2d weight [C][C][k][k] (k = 2s) -> the score kernels' packed bf16 operand (forward or data gradient)."""
    C, _, k, _ = w.shape
    n = int(lib.load().seg_score_packed_elems(C, k // 2))
    if n < 0:
        raise RuntimeError(f"score kernels: C = {C}, k = {k} unsupported (1 <= C <= 160, k = 2s, s <= 8)")
    out = torch.empty(n, dtype=torch.bfloat16, device=w.device)
    call("seg_score_pack", ptr(w.detach().float().contiguous()), ptr(out), C, k // 2, int(bool(bwd)))
    return out


def score_upsample_fwd(x, packed, k, window, skip=None, skip_off=(0, 0), alpha=0.0, bias=None, out_dtype=torch.bfloat16):
    """Window (y0, x0, Ho, Wo) of ConvTranspose2d(C, C, k, k // 2)(x), + alpha * skip[window at skip_off] + bias if skip is
    given.  Returns [N,Ho,Wo,C] of out_dtype; a bf16 result has channel pitch ceil8(C) (pad lanes never written)."""
    N, h, w, C = x.shape
    y0, x0, Ho, Wo = window
    cp = (C + 7) // 8 * 8 if out_dtype == torch.bfloat16 else C
    y = torch.empty((N, Ho, Wo, cp), dtype=out_dtype, device=x.device)[..., :C]
    Hs, Ws = (skip.shape[1], skip.shape[2]) if skip is not None else (0, 0)
    call("seg_score_upsample_fwd", ptr(x), ld(x), N, h, w, C, k // 2, ptr(packed), ptr(y), ld(y),
         DT_BF16 if out_dtype == torch.bfloat16 else DT_F32, y0, x0, Ho, Wo, ptr(skip), ld(skip) if skip is not None else 0, Hs, Ws,
         skip_off[0], skip_off[1], float(alpha), ptr(bias))
    return y


def score_upsample_bwd(dy, packed_bwd, x_shape, k, window):
    """Data gradient [N,h,w,C] bf16 (pitch ceil8(C)) of score_upsample_fwd's transposed conv for the window gradient dy."""
    N, h, w, C = x_shape
    y0, x0, Ho, Wo = window
    assert tuple(dy.shape) == (N, Ho, Wo, C)
    dx = torch.empty((N, h, w, (C + 7) // 8 * 8), dtype=torch.bfloat16, device=dy.device)[..., :C]
    call("seg_score_upsample_bwd", ptr(dy), ld(dy), N, h, w, C, k // 2, ptr(packed_bwd), ptr(dx), ld(dx), y0, x0, Ho, Wo)
    return dx


def score_skip_bwd(dy, skip_shape, skip_off, alpha, out=None):
    """Gradient of the skip map: alpha * dy placed at skip_off, 0 elsewhere (bf16 [N,Hs,Ws,C], pitch ceil8(C) unless `out`)."""
    N, Hs, Ws, C = skip_shape
    if out is None:
        out = torch.empty((N, Hs, Ws, (C + 7) // 8 * 8), dtype=torch.bfloat16, device=dy.device)[..., :C]
    call("seg_score_skip_bwd", ptr(dy), ld(dy), dy.shape[1], dy.shape[2], ptr(out), ld(out), N, Hs, Ws, C, skip_off[0], skip_off[1],
         float(alpha))
    return out


def axpby(x, y, beta):
    call("seg_axpby_bf16", ptr(x), ld(x), ptr(y), ld(y), rows(x), x.shape[-1], float(beta))
    return y


# ---------------------------------------------------------------- input pipeline tail / inference resampling (seg_data.cu)
def resize_nchw(src, Hd, Wd, align_corners=True, flip_x=False, alpha=1.0, out=None, beta=0.0, zoom=False):
    """out = beta*out + alpha * [flip](bilinear resize of fp32 NCHW `src` to Hd x Wd).  zoom=True: scipy.ndimage.zoom(order=1)
    semantics (float64 coordinates, outputs past the last input sample are 0) instead of ATen's."""
    N, C, Hs, Ws = src.shape
    assert src.is_contiguous() and src.dtype == torch.float32
    if out is None:
        out = torch.empty((N, C, Hd, Wd), dtype=torch.float32, device=src.device)
        beta = 0.0
    assert out.is_contiguous() and out.shape == (N, C, Hd, Wd) and out.dtype == torch.float32
    call("seg_resize_nchw_f32", ptr(src), N * C, Hs, Ws, ptr(out), Hd, Wd, 2 if zoom else int(bool(align_corners)), int(flip_x), float(alpha), float(beta))
    return out


def window_add_nchw(src, dst, y0, x0, h, w, flip_x=False, alpha=1.0):
    """dst[:, :, y0:y0+h, x0:x0+w] += alpha * [flip](src)[:, :, :h, :w]"""
    N, C, Hs, Ws = src.shape
    assert src.is_contiguous() and dst.is_contiguous() and src.dtype == dst.dtype == torch.float32 and dst.shape[:2] == (N, C)
    call("seg_window_add_nchw_f32", ptr(src), N * C, Hs, Ws, ptr(dst), dst.shape[2], dst.shape[3], int(y0), int(x0), int(h), int(w),
         int(flip_x), float(alpha))
    return dst


def div_by_count_nchw(x, count_hw):
    N, C, H, W = x.shape
    assert x.is_contiguous() and count_hw.is_contiguous() and count_hw.shape == (H, W) and count_hw.dtype == torch.float32
    call("seg_div_by_count_nchw_f32", ptr(x), N * C, H, W, ptr(count_hw))
    return x


def argmax_nchw(scores):
    N, C, H, W = scores.shape
    assert scores.is_contiguous() and scores.dtype == torch.float32
    labels = torch.empty((N, H, W), dtype=torch.int64, device=scores.device)
    call("seg_argmax_nchw_f32", ptr(scores), N, C, H, W, ptr(labels))
    return labels


def _augment(name, table_bytes, arena, table, taps, B, crop_h, crop_w, mean, std, want_labels, label_map):
    assert arena.dtype == torch.uint8 and table.dtype == torch.uint8 and table.numel() == B * table_bytes
    out = torch.empty((B, 3, crop_h, crop_w), dtype=torch.float32, device=arena.device)
    labels = torch.empty((B, crop_h, crop_w), dtype=torch.int64, device=arena.device) if want_labels else None
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    name = name.replace("_batch_u8", "_mapped_batch_u8") if label_map else name
    head = (ptr(arena), ptr(table)) if taps is None else (ptr(arena), ptr(table), ptr(taps))
    call(name, *head, int(B), int(crop_h), int(crop_w), m3, s3, ptr(out), ptr(labels))
    return out, labels


# label_map=True runs the *_mapped twin of each entry point, which also reads records whose lbl_bytes carries
# lib.AUG_LABEL_MAP (a uint8 label map followed by its 256-entry int32 id table); records without the flag give the same
# output under either kernel.
def augment_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True, label_map=False):
    """arena: uint8 device tensor (images + labels back to back), table: uint8 device tensor of B seg_aug_entry records."""
    return _augment("seg_augment_batch_u8", lib.load().seg_aug_entry_bytes(), arena, table, None, B, crop_h, crop_w, mean, std,
                    want_labels, label_map)


def augment_scale_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True, label_map=False):
    """As augment_batch_u8 with the random-scale resize fused in front; table = B seg_aug_scale_entry records."""
    return _augment("seg_augment_scale_batch_u8", lib.load().seg_aug_scale_entry_bytes(), arena, table, None, B, crop_h, crop_w, mean,
                    std, want_labels, label_map)


def augment_full_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True, label_map=False):
    """augment_scale_batch_u8 with the rotation (cv2.getRotationMatrix2D + warpAffine arithmetic) fused in; table = B
    seg_aug_full_entry records."""
    return _augment("seg_augment_full_batch_u8", lib.load().seg_aug_full_entry_bytes(), arena, table, None, B, crop_h, crop_w, mean,
                    std, want_labels, label_map)


def augment_val_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True, label_map=False):
    """The validation tail (resize so the short side is the crop, centre crop, ToTensor, Normalize) on B seg_aug_scale_entry
    records; each label map in the arena is followed by its PIL NEAREST index tables (x then y, int32)."""
    return _augment("seg_augment_val_batch_u8", lib.load().seg_aug_scale_entry_bytes(), arena, table, None, B, crop_h, crop_w, mean,
                    std, want_labels, label_map)


def augment_full_blur_batch_u8(arena, table, taps, B, crop_h, crop_w, mean, std, want_labels=True, label_map=False):
    """augment_full_batch_u8 with the Gaussian blur after the flip; taps: float32 device tensor [B, 2] of (centre, side)
    taps, (1, 0) for a sample that is not blurred."""
    assert taps.dtype == torch.float32 and taps.is_contiguous() and taps.numel() == 2 * B and taps.device == arena.device
    return _augment("seg_augment_full_blur_batch_u8", lib.load().seg_aug_full_entry_bytes(), arena, table, taps, B, crop_h, crop_w,
                    mean, std, want_labels, label_map)
