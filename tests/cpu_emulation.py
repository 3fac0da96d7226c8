"""TEST-ONLY stand-in for seg_b200.ops: every C-ABI wrapper re-expressed with ATen CPU ops, same signatures and the
same NHWC-bf16 / channel-slice / beta-accumulate conventions.  It exists so the HOST logic of the engine (tape order,
gradient accumulation, concat slices, residual wiring, autograd bridge) can be checked against the oracle on the CPU
box.  It is never imported by the product; tests inject it with monkeypatch.  The real kernels are checked on the GPU
by tests/test_ops_gpu.py and tests/test_model_gpu.py."""
import torch
import torch.nn.functional as F

IMPL_AUTO, IMPL_SIMT, IMPL_TC = 0, 1, 2
ACT_DTYPE = torch.bfloat16  # tests may set this to torch.float32 to take bf16 rounding out of the comparison


def ld(t):
    return t.stride(-2) if t.shape[-2] > 1 else t.shape[-1]


def rows(t):
    m = 1
    for s in t.shape[:-1]:
        m *= s
    return m


def _nchw(t):
    return t.float().permute(0, 3, 1, 2)


def _store(out, val_nhwc, beta=0.0):
    if beta:
        out.copy_((out.float() * beta + val_nhwc).to(out.dtype))
    else:
        out.copy_(val_nhwc.to(out.dtype))
    return out


def _w_oihw(wp, R, S):
    T, K, C = wp.shape
    return wp.float().reshape(R, S, K, C).permute(2, 3, 0, 1).contiguous()


def pack_weight(w, cpad=None):
    K, C, R, S = w.shape
    cpad = cpad or C
    out = torch.zeros(R * S, K, cpad, dtype=ACT_DTYPE)
    out[:, :, :C] = w.detach().permute(2, 3, 0, 1).reshape(R * S, K, C).to(ACT_DTYPE)
    return out


def unpack_wgrad(dwp, shape, beta=0.0, out=None):
    K, C, R, S = shape
    g = dwp[:, :, :C].reshape(R, S, K, C).permute(2, 3, 0, 1)
    if out is None:
        return g.clone()
    out.copy_(out * beta + g if beta else g)
    return out


def new_stats(C, device=None):
    return torch.zeros(2 * C, dtype=torch.float64)


def conv2d_fwd(x, wp, K, R, S, stride=1, pad=0, dil=1, out=None, out_dtype=None, bias=None, beta=0.0, stats=None,
               impl=0, sync=None, sync_ticket=None):
    y = F.conv2d(_nchw(x), _w_oihw(wp, R, S), bias, stride, pad, dil).permute(0, 2, 3, 1)
    if stats is not None:  # fp64 accumulators (zero on entry); sums of the output AS STORED (rounded to the output type),
        C = y.shape[-1]    # which is what bn_apply then normalises
        ys = y.to(out.dtype if out is not None else (out_dtype or ACT_DTYPE)).double()
        stats[:C] += ys.reshape(-1, C).sum(0)
        stats[C:] += (ys * ys).reshape(-1, C).sum(0)
    if out is None:
        out = torch.empty(y.shape, dtype=out_dtype or ACT_DTYPE)
    return _store(out, y, beta)


def conv2d_dgrad(dy, wp, x_shape, R, S, stride=1, pad=0, dil=1, out=None, beta=0.0, impl=0):
    N, H, W, C = x_shape
    g = torch.nn.grad.conv2d_input((N, C, H, W), _w_oihw(wp, R, S), _nchw(dy), stride, pad, dil).permute(0, 2, 3, 1)
    if out is None:
        out = torch.empty(x_shape, dtype=ACT_DTYPE)
        beta = 0.0
    return _store(out, g, beta)


def conv2d_wgrad(dy, x, R, S, stride=1, pad=0, dil=1, out=None, impl=0):
    K, C = dy.shape[-1], x.shape[-1]
    g = torch.nn.grad.conv2d_weight(_nchw(x), (K, C, R, S), _nchw(dy), stride, pad, dil)
    gp = g.permute(2, 3, 0, 1).reshape(R * S, K, C)
    if out is None:
        return gp.contiguous()
    out += gp
    return out


def dw_pack_weight(w_c133):
    C = w_c133.shape[0]
    return w_c133.detach().reshape(C, 9).t().contiguous().float()


def dw_unpack_wgrad(g9, out, beta=0.0):
    g = g9.t().reshape(out.shape)
    out.copy_(out * beta + g if beta else g)
    return out


def _dw_w(w9):
    C = w9.shape[1]
    return w9.t().reshape(C, 1, 3, 3).float()


def dwconv_fwd(x, w9, stride=1, pad=1, dil=1, out=None, stats=None, sync=None, sync_ticket=None):
    C = x.shape[-1]
    y = F.conv2d(_nchw(x), _w_round(_dw_w(w9)), None, stride, pad, dil, groups=C).permute(0, 2, 3, 1)
    if out is None:
        out = torch.empty(y.shape, dtype=ACT_DTYPE)
    if stats is not None:  # sums of y AS STORED (rounded to the output type), as conv2d_fwd
        ys = y.to(out.dtype).double()
        stats[:C] += ys.reshape(-1, C).sum(0)
        stats[C:] += (ys * ys).reshape(-1, C).sum(0)
    return _store(out, y)


def dwconv_bwd_data(dy, w9, x_shape, stride=1, pad=1, dil=1, out=None, beta=0.0):
    N, H, W, C = x_shape
    g = torch.nn.grad.conv2d_input((N, C, H, W), _w_round(_dw_w(w9)), _nchw(dy), stride, pad, dil, groups=C).permute(0, 2, 3, 1)
    if out is None:
        out = torch.empty(x_shape, dtype=ACT_DTYPE)
        beta = 0.0
    return _store(out, g, beta)


def dwconv_bwd_weight(dy, x, stride=1, pad=1, dil=1, out=None, beta=0.0):
    C = x.shape[-1]
    g = torch.nn.grad.conv2d_weight(_nchw(x), (C, 1, 3, 3), _nchw(dy), stride, pad, dil, groups=C).reshape(C, 9).t()
    if out is None:
        return g.contiguous()
    out.copy_(out * beta + g if beta else g)
    return out


def _w_round(w):
    return w  # depthwise taps stay fp32 in the kernels (registers), no bf16 rounding


def im2col(x, R, S, stride, pad, dil, kpad, nchw_f32):
    xn = x.float() if nchw_f32 else _nchw(x)
    N, C, H, W = xn.shape
    cols = F.unfold(xn.to(ACT_DTYPE).float(), (R, S), dil, pad, stride)  # [N, C*R*S, L] ordered (c, r, s)
    P = (H + 2 * pad - dil * (R - 1) - 1) // stride + 1
    Q = (W + 2 * pad - dil * (S - 1) - 1) // stride + 1
    cols = cols.reshape(N, C, R * S, P, Q).permute(0, 3, 4, 2, 1).reshape(N, P, Q, R * S * C)  # (r, s, c)
    out = torch.zeros(N, P, Q, kpad, dtype=ACT_DTYPE)
    out[..., : R * S * C] = cols.to(ACT_DTYPE)
    return out


def bn_stats(x, stats=None, sync=None, sync_ticket=None):
    C = x.shape[-1]
    if stats is None:
        stats = torch.zeros(2 * C, dtype=torch.float64)
    f = x.double().reshape(-1, C)
    stats[:C] += f.sum(0)
    stats[C:] += (f * f).sum(0)
    return stats


def bn_finalize(stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var):
    C = gamma.numel()
    mean = stats[:C].double() / count
    var = (stats[C:].double() / count - mean * mean).clamp(min=0)
    istd = var.clamp(min=eps) ** -0.5 if clamp_eps else (var + eps) ** -0.5
    if running_mean is not None:
        unb = var * count / (count - 1) if count > 1 else var
        running_mean.copy_(((1 - momentum) * running_mean.double() + momentum * mean).float())
        running_var.copy_(((1 - momentum) * running_var.double() + momentum * unb).float())
    sc = gamma.double() * istd
    return torch.cat([sc, beta.double() - mean * sc]).float(), torch.cat([mean, istd]).float()


def bn_eval_scale_shift(gamma, beta, rm, rv, eps, want_save=False):
    istd = (rv + eps).rsqrt()
    ss = torch.cat([gamma * istd, beta - rm * gamma * istd])
    return (ss, torch.cat([rm, istd])) if want_save else ss


def bn_apply(x, ss, res=None, out=None, relu=True, drop_p=0.0, seed=0, step_ctr=None, drop_hw=0):
    C = x.shape[-1]
    v = x.float() * ss[:C] + ss[C:]
    if res is not None:
        v = v + res.float()
    if relu:
        v = v.clamp(min=0)
    assert drop_p == 0.0, "emulation runs with dropout disabled"
    if out is None:
        out = torch.empty(x.shape, dtype=ACT_DTYPE)
    return _store(out, v)


def bn_apply_train(x, stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var, res=None, out=None,
                   relu=True, drop_p=0.0, seed=0, step_ctr=None, drop_hw=0):
    ss, save = bn_finalize(stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var)
    return bn_apply(x, ss, res=res, out=out, relu=relu, drop_p=drop_p, seed=seed, step_ctr=step_ctr), save


def _dz(dout, out, relu, drop_p, x=None, save=None, gamma=None, beta=None):
    dz = dout.float()
    if relu and out is None:  # mask recomputed from x with the forward's coefficients
        C = x.shape[-1]
        sc = gamma * save[C:]
        dz = dz * ((x.float() * sc + (beta - save[:C] * sc)) > 0)
    elif relu:
        dz = dz * (out.float() > 0)
    return dz


def bn_bwd_reduce_acc_words(C):
    return 2 * C + 1


def bn_bwd_reduce(dout, out, x, save, relu=True, drop_p=0.0, dgamma=None, dbeta=None, accumulate=False, acc=None,
                  gamma=None, beta=None, sync=None):
    C = x.shape[-1]
    dz = _dz(dout, out, relu, drop_p, x, save, gamma, beta).reshape(-1, C)
    xhat = ((x.float() - save[:C]) * save[C:]).reshape(-1, C)
    sums = torch.cat([dz.sum(0), (dz * xhat).sum(0)])
    if dgamma is not None:
        bn_param_grad(sums, dgamma, dbeta, accumulate)
    return sums


def bn_bwd_apply(dout, out, x, save, gamma, sums, count, relu=True, drop_p=0.0, dx=None, dres=None, beta_res=0.0, beta=None):
    C = x.shape[-1]
    dz = _dz(dout, out, relu, drop_p, x, save, gamma, beta)
    xhat = (x.float() - save[:C]) * save[C:]
    g = gamma * save[C:] * (dz - sums[:C] / count - xhat * sums[C:] / count)
    if dres is not None:
        _store(dres, dz, beta_res)
    if dx is None:
        dx = torch.empty(x.shape, dtype=ACT_DTYPE)
    return _store(dx, g)


def bn_bwd_fused(dout, out, x, save, gamma, count_total, relu=True, drop_p=0.0, dgamma=None, dbeta=None, accumulate=False,
                 dx=None, dres=None, beta_res=0.0, beta=None, zero_sums=False, tickets=None, sync=None):
    assert sync is None
    sums = bn_bwd_reduce(dout, out, x, save, relu=relu, drop_p=drop_p, dgamma=dgamma, dbeta=dbeta, accumulate=accumulate,
                         gamma=gamma, beta=beta)
    g = torch.zeros_like(sums) if zero_sums else sums
    return bn_bwd_apply(dout, out, x, save, gamma, g, count_total, relu=relu, drop_p=drop_p, dx=dx, dres=dres, beta_res=beta_res,
                        beta=beta), sums


def bn_param_grad(sums, dgamma, dbeta, accumulate=False):
    C = sums.numel() // 2
    if accumulate:
        dbeta += sums[:C]
        dgamma += sums[C:]
    else:
        dbeta.copy_(sums[:C])
        dgamma.copy_(sums[C:])


def maxpool3x3s2_fwd(x):
    y, idx = F.max_pool2d(_nchw(x), 3, 2, 1, return_indices=True)
    return y.permute(0, 2, 3, 1).to(ACT_DTYPE).contiguous(), idx


def maxpool3x3s2_bwd(dy, idx, x_shape):
    N, H, W, C = x_shape
    g = F.max_unpool2d(_nchw(dy), idx, 3, 2, 1, output_size=(H, W))
    # max_unpool assigns (no accumulation on overlapping windows) -> use scatter_add for exactness
    flat = torch.zeros(N, C, H * W)
    flat.scatter_add_(2, idx.reshape(N, C, -1), _nchw(dy).reshape(N, C, -1))
    return flat.reshape(N, C, H, W).permute(0, 2, 3, 1).to(ACT_DTYPE).contiguous()


def adaptive_avgpool_fwd(x, bins):
    return F.adaptive_avg_pool2d(_nchw(x), bins).permute(0, 2, 3, 1).to(ACT_DTYPE).contiguous()


def adaptive_avgpool_bwd(dy, x_shape, bins, dx=None, beta=0.0):
    N, H, W, C = x_shape
    with torch.enable_grad():
        xin = torch.zeros(N, C, H, W, requires_grad=True)
        F.adaptive_avg_pool2d(xin, bins).backward(_nchw(dy))
    if dx is None:
        dx = torch.empty(x_shape, dtype=ACT_DTYPE)
        beta = 0.0
    return _store(dx, xin.grad.permute(0, 2, 3, 1), beta)


def bilinear_fwd(x, Ho, Wo, align_corners, out=None):
    y = F.interpolate(_nchw(x), size=(Ho, Wo), mode="bilinear", align_corners=align_corners).permute(0, 2, 3, 1)
    if out is None:
        out = torch.empty(y.shape, dtype=ACT_DTYPE)
    return _store(out, y)


def bilinear_bwd(dy, Hi, Wi, align_corners, dx=None, beta=0.0):
    N, Ho, Wo, C = dy.shape
    with torch.enable_grad():
        xin = torch.zeros(N, C, Hi, Wi, requires_grad=True)
        F.interpolate(xin, size=(Ho, Wo), mode="bilinear", align_corners=align_corners).backward(_nchw(dy))
    if dx is None:
        dx = torch.empty((N, Hi, Wi, C), dtype=ACT_DTYPE)
        beta = 0.0
    return _store(dx, xin.grad.permute(0, 2, 3, 1), beta)


def bilinear_logits_fwd(x, Ho, Wo, align_corners):
    return F.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=align_corners).contiguous()


def bilinear_logits_bwd(dy, Hi, Wi, align_corners, ldx):
    N, C, Ho, Wo = dy.shape
    with torch.enable_grad():
        xin = torch.zeros(N, C, Hi, Wi, requires_grad=True)
        F.interpolate(xin, size=(Ho, Wo), mode="bilinear", align_corners=align_corners).backward(dy)
    out = torch.zeros(N, Hi, Wi, ldx, dtype=ACT_DTYPE)
    out[..., :C] = xin.grad.permute(0, 2, 3, 1).to(ACT_DTYPE)
    return out


def _unweighted_mean_ce_only(weight, gamma, mean):
    if weight is not None or gamma is not None or not mean:
        raise NotImplementedError("the emulation restates the unweighted mean cross-entropy only")


def loss_nchw_fwd(logits, target, ignore_index, weight=None, gamma=None, mean=True, reduce_fn=None):
    _unweighted_mean_ce_only(weight, gamma, mean)
    valid = target != ignore_index
    loss_sum = F.cross_entropy(logits, target, ignore_index=ignore_index, reduction="sum")
    accum = torch.tensor([loss_sum.item(), float(valid.sum())], dtype=torch.float64)
    if reduce_fn is not None:
        reduce_fn(accum)
    return (accum[0] / accum[1].clamp(min=1)).float(), accum


def loss_nchw_bwd(logits, target, ignore_index, accum, weight=None, gamma=None, mean=True, gscale=None):
    """d(loss sum)/d(logits) / accum.count  (the count may be the cross-rank total)"""
    _unweighted_mean_ce_only(weight, gamma, mean)
    with torch.enable_grad():
        l = logits.detach().clone().requires_grad_(True)
        F.cross_entropy(l, target, ignore_index=ignore_index, reduction="sum").backward()
    return (l.grad / accum[1].clamp(min=1)).float() * (gscale.reshape(()) if gscale is not None else 1.0)


def relu_fwd(x):
    return x.float().clamp(min=0).to(ACT_DTYPE)


def relu_bwd(dy, y, dx, beta):
    return _store(dx, dy.float() * (y.float() > 0), beta)


def counter_add(ctr, inc=1):
    ctr += inc


def axpby(x, y, beta):
    return _store(y, x.float(), beta)
