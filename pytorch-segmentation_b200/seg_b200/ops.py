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
    """(desc pointer, ticket pointer, ticket tensor kept alive) for a SyncBN producer / consumer call."""
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


def bn_bwd_reduce_acc_words(C):
    """fp64 words of the zeroed accumulator block of bn_bwd_reduce: [slots][2C] sums + one ticket word."""
    return int(lib.load().seg_bn_bwd_reduce_slots()) * 2 * C + 1


def bn_bwd_reduce(dout, out, x, save, relu=True, drop_p=0.0, dgamma=None, dbeta=None, accumulate=False, acc=None,
                  gamma=None, beta=None, sync=None):
    """Returns sums fp32 [2C] = (sum dz, sum dz*xhat); optionally writes the parameter gradients from them.  One launch: fp64
    atomics into `acc` (exact, bit-reproducible), the last block rounds / writes.  acc: zeroed fp64 [bn_bwd_reduce_acc_words(C)]
    (accumulator copies + ticket) from the caller's arena, allocated here if None.  sync: SyncBN — the last block pushes the sums to the peers (the
    consumer is bn_bwd_apply(sync=...)).
    out=None (with relu, gamma, beta): the ReLU mask is recomputed from x instead of read from the stored activation."""
    C = x.shape[-1]
    M = rows(x)
    sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    nw = bn_bwd_reduce_acc_words(C)
    if acc is None:
        acc = torch.zeros(nw, dtype=torch.float64, device=x.device)
    assert acc.dtype == torch.float64 and acc.numel() >= nw
    call("seg_bn_bwd_reduce", ptr(dout), ld(dout), ptr(out), ld(out) if out is not None else 0, ptr(x), ld(x), ptr(save),
         M, C, int(relu), float(drop_p), ptr(sums), ptr(acc), acc.data_ptr() + 8 * (nw - 1), ptr(dgamma), ptr(dbeta), int(accumulate),
         ptr(gamma), ptr(beta), ctypes.addressof(sync.desc) if sync is not None else None,
         meta=_meta_rows(M, C, 3 if (relu and out is not None) else 2))
    return sums


def bn_apply_train(x, stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var, res=None, out=None,
                   relu=True, drop_p=0.0, seed=0, step_ctr=None, drop_hw=0, sync=None, sync_done=None):
    """Training-mode BN (+residual, ReLU, dropout) straight from the batch sums.  Returns (out, save[2C]).
    sync (comm.SyncBNGroup, with the producing conv2d_fwd(sync=...)): the kernel waits for the world's flags and adds every
    rank's sums itself; `count` is the world's; sync_done: one zeroed word (allocated here if None)."""
    C = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    save = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    assert stats.dtype == torch.float64
    if sync is not None and sync_done is None:
        sync_done = torch.zeros(1, dtype=torch.float32, device=x.device)
    call("seg_bn_apply_train", ptr(x), ld(x), ptr(stats), float(count), ptr(gamma), ptr(beta), float(eps), float(momentum),
         int(clamp_eps), ptr(running_mean), ptr(running_var), ptr(save), ptr(res), ld(res) if res is not None else 0,
         ptr(out), ld(out), rows(x), C, int(relu), float(drop_p), int(seed), ptr(step_ctr), int(drop_hw),
         ctypes.addressof(sync.desc) if sync is not None else None, ptr(sync_done) if sync is not None else None,
         meta=_meta_rows(rows(x), C, 3 if res is not None else 2, res is not None))
    return out, save


def bn_bwd_apply(dout, out, x, save, gamma, sums, count, relu=True, drop_p=0.0, dx=None, dres=None, beta_res=0.0, beta=None,
                 sync=None, sync_done=None):
    C = x.shape[-1]
    if dx is None:
        dx = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    sp, tp, _keep = _sync_args(sync, sync_done, x.device)
    call("seg_bn_bwd_apply", ptr(dout), ld(dout), ptr(out), ld(out) if out is not None else 0, ptr(x), ld(x), ptr(save),
         ptr(gamma), ptr(sums), float(count), rows(x), C, int(relu), float(drop_p), ptr(dx), ld(dx), ptr(dres),
         ld(dres) if dres is not None else 0, float(beta_res), ptr(beta), sp, tp,
         meta=_meta_rows(rows(x), C, (3 if (relu and out is not None) else 2) + 1 + (0 if dres is None else (2 if beta_res != 0.0 else 1)), dres is not None))
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
                 dx=None, dres=None, beta_res=0.0, beta=None, zero_sums=False, tickets=None, sync=None):
    """BatchNorm backward in ONE cooperative launch (reduce -> grid barrier -> fixed-order cross-block sum [-> SyncBN exchange]
    -> apply).  Returns (dx, local sums [2C]).  out=None: ReLU mask recomputed from x (needs beta).  tickets: 2 zeroed words."""
    C = x.shape[-1]
    M = rows(x)
    if dx is None:
        dx = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    nr, nt = bn_bwd_fused_workspace(M, C)
    fr = torch.empty(max(nr, 1), dtype=torch.float32, device=x.device)
    if tickets is None:
        tickets = torch.zeros(max(nt, 1), dtype=torch.float32, device=x.device)
    call("seg_bn_bwd_fused", ptr(dout), ld(dout), ptr(out), ld(out) if out is not None else 0, ptr(x), ld(x), ptr(save), ptr(gamma),
         ptr(beta), float(count_total), M, C, int(relu), float(drop_p), ptr(sums), ptr(fr), ptr(tickets), ptr(dgamma), ptr(dbeta),
         int(accumulate), ptr(dx), ld(dx), ptr(dres), ld(dres) if dres is not None else 0, float(beta_res), int(zero_sums),
         ctypes.addressof(sync.desc) if sync is not None else None,
         meta=_meta_rows(M, C, (3 if (relu and out is not None) else 2) * 2 + 1 + (0 if dres is None else (2 if beta_res != 0.0 else 1)), dres is not None))
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


# ---------------------------------------------------------------- loss
def ce_nchw_fwd(logits, target, ignore_index, reduce_fn=None):
    """reduce_fn(accum): optional in-place cross-rank sum of the fp64 (loss sum, valid-pixel count) pair before the mean."""
    N, C, H, W = logits.shape
    assert logits.is_contiguous() and logits.dtype == torch.float32 and target.dtype == torch.int64 and target.is_contiguous()
    accum = torch.zeros(2, dtype=torch.float64, device=logits.device)
    call("seg_ce_nchw_fwd", ptr(logits), ptr(target), N, C, H, W, int(ignore_index), ptr(accum))
    if reduce_fn is not None:
        reduce_fn(accum)
    loss = torch.empty((), dtype=torch.float32, device=logits.device)
    call("seg_ce_finalize", ptr(accum), ptr(loss))
    return loss, accum


def ce_nchw_bwd(logits, target, ignore_index, accum, gscale=None):
    N, C, H, W = logits.shape
    dl = torch.empty_like(logits)
    call("seg_ce_nchw_bwd", ptr(logits), ptr(target), N, C, H, W, int(ignore_index), ptr(accum), ptr(gscale), ptr(dl))
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


def upsample_ce_fwd(logits_lo, target, align_corners, ignore_index, want_argmax=False, reduce_fn=None):
    N, Hi, Wi, C = logits_lo.shape
    _, Ho, Wo = target.shape
    assert logits_lo.is_contiguous() and logits_lo.dtype == torch.float32 and target.is_contiguous()
    accum = torch.zeros(2, dtype=torch.float64, device=logits_lo.device)
    am = torch.empty((N, Ho, Wo), dtype=torch.int32, device=logits_lo.device) if want_argmax else None
    call("seg_upsample_ce_fwd", ptr(logits_lo), ptr(target), N, Hi, Wi, Ho, Wo, C, int(align_corners), int(ignore_index),
         ptr(accum), ptr(am))
    if reduce_fn is not None:  # cross-rank sum of the fp64 (loss sum, valid-pixel count) pair: global-batch mean
        reduce_fn(accum)
    loss = torch.empty((), dtype=torch.float32, device=logits_lo.device)
    call("seg_ce_finalize", ptr(accum), ptr(loss))
    return loss, accum, am


def upsample_ce_bwd(logits_lo, target, align_corners, ignore_index, accum, ldx, gscale=None):
    N, Hi, Wi, C = logits_lo.shape
    _, Ho, Wo = target.shape
    dlo = torch.empty((N, Hi, Wi, C), dtype=torch.float32, device=logits_lo.device)
    fixed = torch.empty((N, Hi, Wi, C), dtype=torch.int64, device=logits_lo.device)
    dx = torch.empty((N, Hi, Wi, ldx), dtype=torch.bfloat16, device=logits_lo.device)
    call("seg_upsample_ce_bwd", ptr(logits_lo), ptr(target), N, Hi, Wi, Ho, Wo, C, int(align_corners), int(ignore_index),
         ptr(accum), ptr(gscale), ptr(dlo), ptr(fixed), ptr(dx), ldx)
    return dx, dlo


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


def augment_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True):
    """arena: uint8 device tensor (images + labels back to back), table: uint8 device tensor of B seg_aug_entry records."""
    assert arena.dtype == torch.uint8 and table.dtype == torch.uint8 and table.numel() == B * lib.load().seg_aug_entry_bytes()
    out = torch.empty((B, 3, crop_h, crop_w), dtype=torch.float32, device=arena.device)
    labels = torch.empty((B, crop_h, crop_w), dtype=torch.int64, device=arena.device) if want_labels else None
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    call("seg_augment_batch_u8", ptr(arena), ptr(table), int(B), int(crop_h), int(crop_w), m3, s3, ptr(out), ptr(labels))
    return out, labels


def augment_scale_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True):
    """As augment_batch_u8 with the random-scale resize fused in front; table = B seg_aug_scale_entry records."""
    assert arena.dtype == torch.uint8 and table.dtype == torch.uint8 and table.numel() == B * lib.load().seg_aug_scale_entry_bytes()
    out = torch.empty((B, 3, crop_h, crop_w), dtype=torch.float32, device=arena.device)
    labels = torch.empty((B, crop_h, crop_w), dtype=torch.int64, device=arena.device) if want_labels else None
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    call("seg_augment_scale_batch_u8", ptr(arena), ptr(table), int(B), int(crop_h), int(crop_w), m3, s3, ptr(out), ptr(labels))
    return out, labels


def augment_full_batch_u8(arena, table, B, crop_h, crop_w, mean, std, want_labels=True):
    """augment_scale_batch_u8 with the rotation (cv2.getRotationMatrix2D + warpAffine arithmetic) fused in; table = B
    seg_aug_full_entry records."""
    assert arena.dtype == torch.uint8 and table.dtype == torch.uint8 and table.numel() == B * lib.load().seg_aug_full_entry_bytes()
    out = torch.empty((B, 3, crop_h, crop_w), dtype=torch.float32, device=arena.device)
    labels = torch.empty((B, crop_h, crop_w), dtype=torch.int64, device=arena.device) if want_labels else None
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    call("seg_augment_full_batch_u8", ptr(arena), ptr(table), int(B), int(crop_h), int(crop_w), m3, s3, ptr(out), ptr(labels))
    return out, labels
