"""FCN8 on the H100: the ReLU + ceil-mode 2x2 max-pool kernels bit for bit against ATen's CUDA F.max_pool2d(F.relu(x), 2, 2,
ceil_mode=True, return_indices=True) and its autograd, the ReLU + dropout kernels, the class-map transposed-convolution
kernels against a float64 per-element bound in the style of tests/conv_check.py, the model against the fp32 oracle of
oracle/fcn.py (pinned to the reference by tests/golden/fcn.npz) with bounds set by an ATen bf16 run of the same model, and
FusedTrainStep and the plugin surface on the model."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import conv_check as cc
import loss_check as lc
from oracle import fcn as ofc
from oracle import losses as ol
from oracle import models as om
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import lib, losses, ops
    from seg_b200.lib import DT_BF16, DT_F32, ptr
    from seg_b200.train import FusedTrainStep

DEV = "cuda"
F32, BF16, U8, I16 = torch.float32, torch.bfloat16, torch.uint8, torch.int16
CODE_SENTINEL = 0xA5


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_cap():
    """Vectors one pass of an elementwise kernel's grid covers: grid_for's cap (8 blocks of 256 threads per SM)."""
    return sms() * 8 * 256


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "fcn.txt"), "a")

    def write(line):
        print(line)
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def guarded(shape, dtype):
    """A dense tensor of `shape` followed by one sentinel guard image: (buffer [N + 1, ...], view of the first N)."""
    buf = torch.empty((shape[0] + 1,) + tuple(shape[1:]), dtype=dtype, device=DEV)
    if dtype == U8:
        buf.fill_(CODE_SENTINEL)
    else:
        cc.sentinel_fill(buf)
    return buf, buf[: shape[0]]


def check_guard(case, buf, dtype):
    g = buf[-1]
    ok = (g == CODE_SENTINEL).all() if dtype == U8 else cc.is_sentinel(g.cpu()).all()
    assert bool(ok), f"{case}: the guard image after the output was overwritten"


def bits(t):
    return t.view(I16) if t.dtype == BF16 else t


# ------------------------------------------------------------------------------------------------ ReLU + ceil-mode pool
def make_pool_input(N, H, W, C, seed):
    """bf16 NHWC raw conv outputs with planted cases: ties with the maximum, all-negative windows, all-zero windows, ±inf
    and NaNs (one or two per window: the last one wins)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, C, generator=g).bfloat16().float()
    sel = torch.rand(N, H, W, C, generator=g)
    x[sel < 0.02] = float("nan")
    x[(sel > 0.02) & (sel < 0.03)] = float("inf")
    x[(sel > 0.03) & (sel < 0.05)] = float("-inf")
    x[(sel > 0.05) & (sel < 0.08)] = 0.0
    P, Q = H // 2, W // 2
    if P and Q:
        win = x[:, : 2 * P, : 2 * Q].reshape(N, P, 2, Q, 2, C).clone()
        s2 = torch.rand(N, P, Q, C, generator=g)
        m = win.amax((2, 4))
        win[:, :, 1, :, 0][s2 < 0.2] = m[s2 < 0.2]                      # tie with the maximum, later in the window
        neg = (s2 > 0.3) & (s2 < 0.45)                                  # every element <= 0: the pooled value is 0
        for r in (0, 1):
            for t in (0, 1):
                win[:, :, r, :, t][neg] = -win[:, :, r, :, t][neg].abs()
        x[:, : 2 * P, : 2 * Q] = win.reshape(N, 2 * P, 2 * Q, C)
    x[x == 0] = 0.0  # no negative zeros: relu(-0.0) may be either sign in ATen
    return x.bfloat16().to(DEV)


def run_pool(x, dy):
    N, H, W, C = x.shape
    P, Q = (H + 1) // 2, (W + 1) // 2
    yb, y = guarded((N, P, Q, C), BF16)
    cb, code = guarded((N, P, Q, C), U8)
    lib.call("seg_relu_maxpool2x2_ceil_fwd", ptr(x), ptr(y), ptr(code), N, H, W, C)
    dxb, dx = guarded((N, H, W, C), BF16)
    lib.call("seg_relu_maxpool2x2_ceil_bwd", ptr(dy), ptr(code), ptr(dx), N, H, W, C)
    torch.cuda.synchronize()
    return (y, code, dx), (yb, cb, dxb)


def pool_case(log, N, H, W, C, seed):
    case = f"relu+maxpool2x2 ceil {N}x{H}x{W}x{C}"
    x = make_pool_input(N, H, W, C, seed)
    P, Q = (H + 1) // 2, (W + 1) // 2
    dy = torch.randn(N, P, Q, C, generator=torch.Generator().manual_seed(seed + 1)).bfloat16().to(DEV)
    (y, code, dx), guards = run_pool(x, dy)
    for buf, dt, what in zip(guards, (BF16, U8, BF16), ("y", "code", "dx")):
        check_guard(f"{case} {what}", buf, dt)
    xr = x.permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    ry, ridx = F.max_pool2d(F.relu(xr), 2, 2, ceil_mode=True, return_indices=True)
    ry.backward(dy.permute(0, 3, 1, 2).contiguous())
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    ry, ridx, rdx = nhwc(ry.detach()), nhwc(ridx), nhwc(xr.grad)
    assert torch.equal(bits(y), bits(ry)), f"{case}: pooled values differ from ATen's"
    assert torch.equal(bits(dx), bits(rdx)), f"{case}: gradient differs from ATen's relu + pool autograd"
    live = (ry.float() > 0) | torch.isnan(ry.float())
    assert code.max().item() <= 7 and torch.equal(code >= 4, ~live), f"{case}: dead-window flags wrong"
    p = torch.arange(P, device=DEV).view(1, P, 1, 1)
    q = torch.arange(Q, device=DEV).view(1, 1, Q, 1)
    c = (code & 3).long()
    idx = (2 * p + c // 2) * W + 2 * q + c % 2
    assert torch.equal(idx[live], ridx[live]), f"{case}: codes differ from ATen's indices where the max is > 0 or NaN"
    again, _ = run_pool(x, dy)
    for a, b, what in zip((y, code, dx), again, ("y", "code", "dx")):
        assert torch.equal(bits(a), bits(b)), f"{case}: {what} not bit-reproducible"
    log(f"{case}: bit-identical to ATen (values, gradient, codes of {int(live.sum())} live windows); "
        f"NaN inputs {int(torch.isnan(x.float()).sum())}, pooled vectors {N * P * Q * C // 8} (grid cap {grid_cap()})")


@pytest.mark.parametrize("C", [8, 64, 512])
@pytest.mark.parametrize("hw", [(1, 1), (1, 2), (2, 1), (2, 2), (3, 3), (1, 7), (3, 8), (17, 23), (50, 75), (25, 37)])
def test_relu_pool_ceil_matches_aten(log, hw, C):
    pool_case(log, 2, hw[0], hw[1], C, seed=hw[0] * 131 + hw[1] + C)


@pytest.mark.parametrize("extra", [-1, 0, 1])
def test_relu_pool_ceil_at_the_grid_cap(log, extra):
    """N * P * Q * C / 8 = SMs * 8 * 256 + extra pooled vectors, H odd: the last window row is partial."""
    n = grid_cap() + extra
    pool_case(log, 1, 2 * n - 1, 3, 8, seed=40 + extra)


def test_relu_pool_ceil_several_grid_strides(log):
    pool_case(log, 1, 2 * (3 * grid_cap() + 5) - 1, 1, 8, seed=45)
    pool_case(log, 2, 2 * (grid_cap() // 64) + 1, 2 * 3 + 1, 64, seed=46)


def test_relu_pool_ceil_rejects_bad_channels():
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.relu_maxpool2x2_ceil_fwd(torch.zeros(1, 4, 4, 12, dtype=BF16, device=DEV))


# ------------------------------------------------------------------------------------------------ ReLU + dropout
def test_relu_dropout(log):
    M, C = 4096, 512
    x = torch.randn(M, C, generator=torch.Generator().manual_seed(3)).bfloat16().to(DEV)
    y0 = ops.relu_dropout_fwd(x, 0.0)
    assert torch.equal(bits(y0), bits(ops.relu_fwd(x))), "p = 0 is not ReLU"
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    p = 0.5
    y1 = ops.relu_dropout_fwd(x, p, seed=7, step_ctr=ctr)
    assert torch.equal(bits(y1), bits(ops.relu_dropout_fwd(x, p, seed=7, step_ctr=ctr))), "not bit-reproducible"
    pos = x.float() > 0
    kept = y1.float() != 0
    want = (F.relu(x.float()) / (1 - p)).bfloat16()
    assert torch.equal(bits(y1[kept]), bits(want[kept])), "kept elements differ from relu / (1 - p)"
    assert not (kept & ~pos).any()
    n = int(pos.sum())
    frac = 1 - int(kept.sum()) / n
    sigma = math.sqrt(p * (1 - p) / n)
    log(f"relu+dropout p={p}: dropped fraction {frac:.5f} of {n} positive elements (5 sigma = {5 * sigma:.5f})")
    assert abs(frac - p) < 5 * sigma
    ops.counter_add(ctr, 1)
    y2 = ops.relu_dropout_fwd(x, p, seed=7, step_ctr=ctr)
    overlap = ((y2.float() != 0) & kept).sum().item() / max(1, int(kept.sum()))
    assert not torch.equal(bits(y1), bits(y2)) and abs(overlap - (1 - p)) < 0.05, "the mask did not change with the step"
    # backward: the keep mask from out > 0
    dy = torch.randn(M, C, generator=torch.Generator().manual_seed(4)).bfloat16().to(DEV)
    dxb, dx = guarded((M, C), BF16)
    ops.relu_dropout_bwd(dy, y1, p, dx, 0.0)
    torch.cuda.synchronize()
    check_guard("relu+dropout bwd", dxb, BF16)
    want = torch.where(y1.float() > 0, dy.float() / (1 - p), torch.zeros_like(dy.float())).bfloat16()
    assert torch.equal(bits(dx), bits(want))


def test_dropout_masks_stay_fresh_under_graph_replay():
    x = torch.randn(512, 256, generator=torch.Generator().manual_seed(5)).bfloat16().to(DEV)
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    out = torch.empty_like(x)
    ops.relu_dropout_fwd(x, 0.5, seed=9, step_ctr=ctr)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.counter_add(ctr, 1)
        out.copy_(ops.relu_dropout_fwd(x, 0.5, seed=9, step_ctr=ctr))
    masks = []
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        masks.append(out.float() != 0)
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])


# ------------------------------------------------------------------------------------------------ score upsampler kernels
def _pitched_input(N, H, W, C, seed, lead=8):
    """bf16-exact values in a channel-pitched buffer whose other lanes hold NaN (the kernels must not read them)."""
    g = torch.Generator().manual_seed(seed)
    v = (torch.randn(N, H, W, C, generator=g)).bfloat16()
    pitch = lead + (C + 7) // 8 * 8 + 8
    buf = torch.full((N, H, W, pitch), float("nan"), dtype=BF16)
    buf[..., lead:lead + C] = v
    return v.double(), buf.to(DEV)[..., lead:lead + C]


def _weight(C, k, seed, dense):
    if dense:
        w = torch.randn(C, C, k, k, generator=torch.Generator().manual_seed(seed)) / math.sqrt(C)
    else:
        w = ofc.upsampling_weight(C, k)
    return w.bfloat16().float()  # the kernels multiply bf16 weights: bound against the bf16-rounded values


def score_fwd_ref(x, w, s, window, skip=None, skip_off=(0, 0), alpha=0.0, bias=None):
    y0, x0, Ho, Wo = window
    xd, wd = x.permute(0, 3, 1, 2), w.double()
    conv = F.conv_transpose2d(xd, wd, stride=s)[:, :, y0:y0 + Ho, x0:x0 + Wo].permute(0, 2, 3, 1)
    mag = F.conv_transpose2d(xd.abs(), wd.abs(), stride=s)[:, :, y0:y0 + Ho, x0:x0 + Wo].permute(0, 2, 3, 1)
    ref, extra = conv.clone(), torch.zeros_like(conv)
    if skip is not None:
        t = alpha * skip[:, skip_off[0]:skip_off[0] + Ho, skip_off[1]:skip_off[1] + Wo]
        if bias is not None:
            t = t + bias.double()
        ref += t
        extra += t.abs() + (bias.double().abs() if bias is not None else 0)
    C = w.shape[0]
    return cc.Ref(ref, ref.clone(), mag, extra, 4 * ((C + 15) // 16 * 16), ("n", "h", "w", "c"))


def score_bwd_ref(dy, w, s, x_shape, window):
    N, h, w_, C = x_shape
    y0, x0, Ho, Wo = window
    g = torch.zeros(N, C, (h + 1) * s, (w_ + 1) * s, dtype=torch.float64)
    g[:, :, y0:y0 + Ho, x0:x0 + Wo] = dy.permute(0, 3, 1, 2)
    ref = F.conv2d(g, w.double(), stride=s).permute(0, 2, 3, 1)
    mag = F.conv2d(g.abs(), w.double().abs(), stride=s).permute(0, 2, 3, 1)
    k = 2 * s
    return cc.Ref(ref, ref.clone(), mag, torch.zeros_like(ref), k * k * ((C + 15) // 16 * 16), ("n", "h", "w", "c"))


def score_case(log, N, h, w, C, k, window, skip_off=None, alpha=0.0, out_f32=False, dense=True, seed=0):
    s = k // 2
    y0, x0, Ho, Wo = window
    case = f"score k={k} C={C} {N}x{h}x{w} window {window}" + (f" skip@{skip_off}" if skip_off else "")
    x, xd = _pitched_input(N, h, w, C, seed)
    wt = _weight(C, k, seed + 1, dense)
    wf, wb = ops.score_pack(wt.to(DEV), False), ops.score_pack(wt.to(DEV), True)
    skip = skd = bias = None
    Hs = Ws = 0
    if skip_off is not None:
        Hs, Ws = skip_off[0] + Ho + 3, skip_off[1] + Wo + 2
        skip, skd = _pitched_input(N, Hs, Ws, C, seed + 2)
        bias = torch.randn(C, generator=torch.Generator().manual_seed(seed + 3)) * 0.1
    r = score_fwd_ref(x, wt, s, window, skip, skip_off or (0, 0), alpha, bias)
    dt = F32 if out_f32 else BF16
    outs = []
    for _ in range(2):
        g = cc.Guarded(N, Ho, Wo, C, dt, cc.GUARD, cc.GUARD, device=DEV)
        lib.call("seg_score_upsample_fwd", ptr(xd), ops.ld(xd), N, h, w, C, s, ptr(wf), ptr(g.view), ops.ld(g.view),
                 DT_F32 if out_f32 else DT_BF16, y0, x0, Ho, Wo, ptr(skd), ops.ld(skd) if skd is not None else 0, Hs, Ws,
                 *(skip_off or (0, 0)), float(alpha), ptr(bias.to(DEV) if bias is not None else None))
        torch.cuda.synchronize()
        cc.check_guards(case + " fwd", g.buf, g.guard_mask())
        cc.check_written(case + " fwd", g.view)
        outs.append(g.view.clone())
    uf = cc.check_elements(case + " fwd", outs[0], r, not out_f32)
    assert torch.equal(bits(outs[0]), bits(outs[1])), f"{case}: forward not bit-reproducible"

    dy, dyd = _pitched_input(N, Ho, Wo, C, seed + 4)
    r = score_bwd_ref(dy, wt, s, (N, h, w, C), window)
    outs = []
    for _ in range(2):
        g = cc.Guarded(N, h, w, C, BF16, cc.GUARD, cc.GUARD, device=DEV)
        lib.call("seg_score_upsample_bwd", ptr(dyd), ops.ld(dyd), N, h, w, C, s, ptr(wb), ptr(g.view), ops.ld(g.view), y0, x0,
                 Ho, Wo)
        torch.cuda.synchronize()
        cc.check_guards(case + " bwd", g.buf, g.guard_mask())
        cc.check_written(case + " bwd", g.view)
        outs.append(g.view.clone())
    ub = cc.check_elements(case + " bwd", outs[0], r, True)
    assert torch.equal(bits(outs[0]), bits(outs[1])), f"{case}: data gradient not bit-reproducible"
    if skip_off is not None:  # d(skip) = alpha * dY at the window, 0 elsewhere
        g = cc.Guarded(N, Hs, Ws, C, BF16, cc.GUARD, cc.GUARD, device=DEV)
        ops.score_skip_bwd(dyd, (N, Hs, Ws, C), skip_off, alpha, out=g.view)
        torch.cuda.synchronize()
        cc.check_guards(case + " skip bwd", g.buf, g.guard_mask())
        want = torch.zeros(N, Hs, Ws, C, dtype=torch.float64)
        want[:, skip_off[0]:skip_off[0] + Ho, skip_off[1]:skip_off[1] + Wo] = alpha * dy
        assert torch.equal(bits(g.view), bits(want.float().bfloat16().to(DEV))), f"{case}: skip gradient"
    log(f"{case}: usage fwd={uf:.4f} bwd={ub:.4f}")


@pytest.mark.parametrize("C", [1, 2, 19, 21, 150, 160])
@pytest.mark.parametrize("k", [4, 16])
def test_score_kernels_dense_weights(log, C, k):
    s = k // 2
    h, w = 5, 7
    score_case(log, 2, h, w, C, k, (3, 1, (h + 1) * s - 5, (w + 1) * s - 2), seed=C * 7 + k)
    score_case(log, 1, h, w, C, k, (0, 0, (h + 1) * s, (w + 1) * s), skip_off=(5, 9), alpha=0.01, seed=C * 7 + k + 50)


def fcn_windows(H, W):
    """(pool5-path class map size, s2 / s4 skip map sizes) of FCN8 at an H x W input."""
    def pool(v):
        return (v + 1) // 2
    h, w = H + 198, W + 198
    sizes = []
    for _ in range(5):
        h, w = pool(h), pool(w)
        sizes.append((h, w))
    return (sizes[4][0] - 6, sizes[4][1] - 6), sizes[3], sizes[2]


@pytest.mark.parametrize("HW", [(64, 64), (50, 75), (512, 512), (513, 513)])
@pytest.mark.parametrize("C", [21, 150])
def test_score_kernels_fcn8_windows(log, HW, C):
    """The three upsamplers of FCN8 at its windows: s2 (skip at 5, alpha 0.01), s4 (skip at 9, alpha 1e-4) in bf16 and the
    cropped fp32 logits, with the bilinear weights."""
    H, W = HW
    (h, w), p4, p3 = fcn_windows(H, W)
    N = 2 if H < 100 else 1
    h2, w2 = 2 * h + 2, 2 * w + 2
    h4, w4 = 2 * h2 + 2, 2 * w2 + 2
    assert 5 + h2 <= p4[0] and 9 + h4 <= p3[0] and 31 + H <= 8 * (h4 + 1)
    score_case(log, N, h, w, C, 4, (0, 0, h2, w2), skip_off=(5, 5), alpha=0.01, dense=False, seed=H + C)
    score_case(log, N, h2, w2, C, 4, (0, 0, h4, w4), skip_off=(9, 9), alpha=1e-4, dense=False, seed=H + C + 1)
    score_case(log, N, h4, w4, C, 16, (31, 31, H, W), out_f32=True, dense=False, seed=H + C + 2)


def test_score_kernels_reject_bad_shapes():
    x = torch.zeros(1, 4, 4, 168, dtype=BF16, device=DEV)
    with pytest.raises(RuntimeError, match="160"):
        ops.score_pack(torch.zeros(161, 161, 4, 4, device=DEV), False)
    with pytest.raises(RuntimeError, match="C <= 160"):  # the C entry point's own check
        lib.call("seg_score_upsample_fwd", ptr(x), 168, 1, 4, 4, 161, 2, ptr(x), ptr(x), 168, DT_BF16, 0, 0, 4, 4, None, 0, 0, 0,
                 0, 0, 0.0, None)
    wp = ops.score_pack(torch.zeros(8, 8, 4, 4, device=DEV), False)
    with pytest.raises(RuntimeError, match="outside"):
        ops.score_upsample_fwd(x[..., :8], wp, 4, (0, 0, 11, 10))


# ------------------------------------------------------------------------------------------------ the model
_SD = {}


def state_dict(nc, seed, dense_up=False):
    key = (nc, seed, dense_up)
    if key not in _SD:
        _SD[key] = ofc.fcn8_state_dict(nc, seed=seed, dense_up=dense_up)
    return _SD[key]


def _model(seed, nc=7, dropout=True, dense_up=False):
    m = seg_b200.FCN8(nc, pretrained=False)
    m.load_state_dict(state_dict(nc, seed, dense_up), strict=True)
    m.engine_dropout = dropout
    return m.cuda().train()


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def cosine(a, b):
    return F.cosine_similarity(a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten(), dim=0).item()


def bf16_control(sd, x, y):
    """The oracle's forward and backward run by ATen on the GPU in bf16: the error a plain bf16 implementation of the same
    model makes.  Returns (logits fp32 CPU, {name: grad})."""
    bsd = {k: v.to(DEV, BF16) for k, v in sd.items()}
    for k, v in bsd.items():
        if not k.startswith("up_"):
            v.requires_grad_(True)
    out = ofc.fcn8_forward(bsd, x.to(DEV, BF16))
    loss = F.cross_entropy(out.float(), y.to(DEV), ignore_index=255)
    loss.backward()
    return out.detach().float().cpu(), {k: v.grad.float().cpu() for k, v in bsd.items() if v.grad is not None}


BOUND_FACTOR = 4.0  # the engine may be this many times further from the fp32 oracle than the ATen bf16 run is


@pytest.mark.parametrize("dense_up", [False, True], ids=["bilinear_up", "dense_up"])
@pytest.mark.parametrize("hw", [(64, 64), (50, 75)], ids=["64x64", "50x75"])
def test_train_step_parity(log, hw, dense_up):
    """Every forward and backward kernel in context against the fp32 oracle (dropout off), with the logits bound and the
    gradient-direction bound set from an ATen bf16 run of the same model."""
    nc = 21
    sd = state_dict(nc, 11, dense_up)
    m = _model(11, nc, dropout=False, dense_up=dense_up)
    x, y = synth.make_batch(2, hw[0], hw[1], nc, 255, seed=9061)
    osd = om.clone_sd(sd, requires_grad=True)
    for name, _ in ofc.UPSAMPLERS:
        osd[name + ".weight"].requires_grad_(False)
    ref = ofc.fcn8_forward(osd, x)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    ctrl_out, ctrl_grads = bf16_control(sd, x, y)
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[fcn8 {hw[0]}x{hw[1]} {'dense' if dense_up else 'bilinear'} upsamplers]"
    e, ec = relerr(out, ref), relerr(ctrl_out, ref)
    log(f"{tag} logits rel_err vs fp32 oracle {e:.3e} (ATen bf16 {ec:.3e}); loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert out.shape == ref.shape == (2, nc) + hw and e <= BOUND_FACTOR * ec
    cos, ccos = {}, {}
    for name, p in m.named_parameters():
        if not p.requires_grad:
            assert p.grad is None, name
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        cos[name] = cosine(p.grad, osd[name].grad)
        ccos[name] = cosine(ctrl_grads[name], osd[name].grad)
    worst, cworst = min(cos, key=cos.get), min(ccos, key=ccos.get)
    log(f"{tag} grads vs fp32 oracle: min cosine {cos[worst]:.5f} at {worst} (ATen bf16 {ccos[cworst]:.5f} at {cworst})")
    assert 1 - cos[worst] <= BOUND_FACTOR * (1 - ccos[cworst]), (cos[worst], worst, ccos[cworst], cworst)
    m.eval()
    with torch.no_grad():
        ev = m(x.cuda())
    assert relerr(ev, ofc.fcn8_forward(osd, x)) <= BOUND_FACTOR * ec


def _crit(name, C):
    if name == "ce":
        return losses.CrossEntropyLoss2d(ignore_index=255)
    if name == "wce":
        return losses.CrossEntropyLoss2d(weight=lc.weights(C, 5).cuda(), ignore_index=255)
    return losses.FocalLoss(ignore_index=255)


@pytest.mark.parametrize("name", ["ce", "wce", "focal"])
def test_fused_step_first_loss_and_counters_equal_plugin(log, name):
    x, y = synth.make_batch(2, 50, 75, 7, 255, seed=9063)
    xd, yd = x.cuda(), y.cuda()
    crit = _crit(name, 7)
    with torch.no_grad():
        out = _model(41)(xd)
        ref = float(crit(out, yd))
        want = ops.eval_metrics_nchw(out, yd, 7)
    s = FusedTrainStep(_model(41), lr=0.005, loss=crit, metrics=True)
    got = float(s.step(xd, yd))
    log(f"fused step [fcn8 {name} 50x75] first loss {got:.7f}, plugin {ref:.7f}")
    assert abs(got - ref) <= 1e-5 * abs(ref)
    assert torch.equal(s.seg_counters, want)


def test_fused_step_graph_replay_is_bit_identical():
    """Dropout off: the graph path's two warm-up steps advance the device step counter, so its masks are a later draw of
    the same stream (test_dropout_masks_stay_fresh_under_graph_replay covers the masks under replay)."""
    x, y = synth.make_batch(2, 50, 75, 7, 255, seed=9064)
    xd, yd = x.cuda(), y.cuda()
    se = FusedTrainStep(_model(42, dropout=False), lr=0.005, metrics=True)
    sg = FusedTrainStep(_model(42, dropout=False), lr=0.005, metrics=True, cuda_graph=True)
    for i in range(3):
        le, lg = float(se.step(xd, yd)), float(sg.step(xd, yd))
        assert le == le and le == lg, (i, le, lg)
        assert torch.equal(se.seg_counters, sg.seg_counters)
    assert torch.equal(se.flat_grad, sg.flat_grad)
    for (n, a), (_, b) in zip(se.model.state_dict().items(), sg.model.state_dict().items()):
        assert torch.equal(a, b), n
    sg.release_graph()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_evaluate_changes_no_training_state(graph):
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9065)
    xd, yd = x.cuda(), y.cuda()
    s = FusedTrainStep(_model(43), lr=0.005, metrics=True, cuda_graph=graph)
    s.step(xd, yd)
    m = s.model
    before = ([t.clone() for t in m.state_dict().values()], s.flat_mom.clone(), m._step_ctr.clone(), s.steps, m.training)
    s.reset_metrics()
    loss = float(s.evaluate(xd, yd))
    after = ([t.clone() for t in m.state_dict().values()], s.flat_mom.clone(), m._step_ctr.clone(), s.steps, m.training)
    assert all(torch.equal(a, b) for a, b in zip(before[0], after[0]))
    assert torch.equal(before[1], after[1]) and torch.equal(before[2], after[2]) and before[3:] == after[3:]
    m.eval()
    with torch.no_grad():
        out = m(xd)
    m.train()
    assert torch.equal(s.seg_counters, ops.eval_metrics_nchw(out, yd, 7))
    ref = float(losses.CrossEntropyLoss2d(ignore_index=255)(out, yd))
    assert abs(loss - ref) <= 1e-5 * abs(ref)
    if graph:
        s.release_graph()


def test_plugin_surface_graphs():
    """model.cuda_graphs() (dropout off, so every step draws the same masks): the replayed plugin step gives the eager
    step's output and gradients bit for bit; the frozen upsamplers get no gradient."""
    x, y = synth.make_batch(2, 50, 75, 7, 255, seed=9066)
    xd, yd = x.cuda(), y.cuda()
    m = _model(45, dropout=False).cuda_graphs(True, warmup=1)
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    res = []
    for _ in range(4):  # eager (warm-up), capture, replay, replay
        for p in m.parameters():
            p.grad = None
        out = m(xd)
        loss = crit(out, yd)
        loss.backward()
        res.append((out.detach().clone(), loss.detach().clone(), [p.grad for p in m.parameters()]))
    assert m._graph_entries, "no graph was captured"
    for o, l, g in res[1:]:
        assert torch.equal(o, res[0][0]) and torch.equal(l, res[0][1])
        assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(g, res[0][2]))
    assert all((g is None) == n.startswith("up_") for (n, _), g in zip(m.named_parameters(), res[0][2]))
    m.cuda_graphs(False)


@pytest.mark.parametrize("name", ["dice", "ce_dice", "lovasz"])
def test_plugin_losses_backpropagate(log, name):
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9067)
    y[y == 255] = 0  # the Dice losses take no ignore_index
    m = _model(46)
    crit = {"dice": losses.DiceLoss(), "ce_dice": losses.CE_DiceLoss(), "lovasz": losses.LovaszSoftmax()}[name]
    out = m(x.cuda())
    loss = crit(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    log(f"plugin loss [fcn8 {name}] {loss.item():.6f}")
    assert loss.item() == loss.item()
    for n, p in m.named_parameters():
        assert (p.grad is None) == n.startswith("up_"), n
        assert p.grad is None or torch.isfinite(p.grad).all(), n


def test_bad_inputs_raise_before_any_launch():
    m = _model(47)
    n = lib.launch_count()
    with pytest.raises(ValueError, match="3-channel"):
        m(torch.zeros(1, 4, 64, 64, device=DEV))
    m.up_output.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="upsampling weight"):
        m(torch.zeros(1, 3, 64, 64, device=DEV))
    assert lib.launch_count() == n


@pytest.mark.parametrize("nc", [21, 150])
@pytest.mark.parametrize("size", [512, 513])
def test_full_size_graph_step(log, size, nc):
    """Graph-replayed 8 x 3 x size^2 fused steps (the configs' crop and batch) have finite losses."""
    x, y = synth.make_batch(8, size, size, nc, 255, seed=9068)
    s = FusedTrainStep(_model(48, nc=nc), lr=0.01, cuda_graph=True)
    losses_ = [float(s.step(x.cuda(), y.cuda())) for _ in range(3)]
    torch.cuda.synchronize()
    log(f"[fcn8 {nc} classes 8x3x{size}x{size} graph step] losses " + " ".join(f"{v:.6f}" for v in losses_))
    assert all(v == v and abs(v) < 1e3 for v in losses_)
    s.release_graph()
