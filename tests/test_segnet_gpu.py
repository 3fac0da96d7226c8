"""SegNet on the H100: the 2x2 max-pool / max-unpool kernels bit for bit against ATen's CUDA F.max_pool2d(2, 2,
return_indices=True) / F.max_unpool2d and their autograd, the classifier conv (3x3, 64 -> 19, bias, fp32 output) against
tests/conv_check.py's per-element float64 bound, the model against the fp32 oracle of oracle/segnet.py (pinned to the
reference by tests/golden/segnet.npz) with bounds set by an ATen bf16 run of the same model, and FusedTrainStep and the
plugin surface on the model."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

import conv_check as cc
import loss_check as lc
from oracle import losses as ol
from oracle import models as om
from oracle import segnet as osn
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import lib, losses, ops
    from seg_b200.lib import IMPL_AUTO, IMPL_TC, ptr
    from seg_b200.train import FusedTrainStep
else:  # keep collection working without a GPU
    IMPL_AUTO, IMPL_TC = 0, 2

DEV = "cuda"
F32, BF16, U8, I16 = torch.float32, torch.bfloat16, torch.uint8, torch.int16
CODE_SENTINEL = 0xA5


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_cap():
    """Vectors one pass of a pooling kernel's grid covers: grid_for's cap (8 blocks of 256 threads per SM)."""
    return sms() * 8 * 256


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "segnet.txt"), "a")

    def write(line):
        print(line)
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


# ------------------------------------------------------------------------------------------------ pool / unpool kernels
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


def make_pool_input(N, H, W, C, seed):
    """bf16 NHWC values with planted cases: ReLU zeros (all-zero windows), exact ties inside windows, -inf windows and NaNs
    (one or two per window: the last one wins)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, C, generator=g)
    x = torch.where(torch.rand(N, H, W, C, generator=g) < 0.3, x.clamp_min(0), x)  # ReLU output: many all-zero windows
    x = x.bfloat16().float()
    P, Q = H // 2, W // 2
    if P and Q:
        win = x[:, : 2 * P, : 2 * Q].reshape(N, P, 2, Q, 2, C).clone()
        sel = torch.rand(N, P, Q, C, generator=g)
        m = win.amax((2, 4))
        win[:, :, 1, :, 0][sel < 0.15] = m[sel < 0.15]                 # tie with the maximum, later in the window
        win[:, :, 0, :, 1][sel < 0.05] = m[sel < 0.05]                 # three-way ties
        zero = (sel > 0.95) & (sel < 0.96)                             # the whole window zero
        for r in (0, 1):
            for t in (0, 1):
                win[:, :, r, :, t][zero] = 0.0
        ninf = (sel > 0.96) & (sel < 0.97)
        for r in (0, 1):
            for t in (0, 1):
                win[:, :, r, :, t][ninf] = float("-inf")             # an all -inf window
        win[:, :, 1, :, 1][(sel > 0.97) & (sel < 0.98)] = float("-inf")
        win[:, :, 0, :, 1][(sel > 0.98) & (sel < 0.99)] = float("nan")
        two = sel > 0.99
        win[:, :, 0, :, 0][two] = float("nan")
        win[:, :, 1, :, 1][two] = float("nan")
        x[:, : 2 * P, : 2 * Q] = win.reshape(N, 2 * P, 2 * Q, C)
    return x.bfloat16().to(DEV)


def run_ours(x, dy, dyu):
    """The four entry points, each into a guarded output; returns (y, code, dx, u, du) and the guard buffers."""
    N, H, W, C = x.shape
    P, Q = H // 2, W // 2
    yb, y = guarded((N, P, Q, C), BF16)
    cb, code = guarded((N, P, Q, C), U8)
    lib.call("seg_maxpool2x2_fwd", ptr(x), ptr(y), ptr(code), N, H, W, C)
    dxb, dx = guarded((N, H, W, C), BF16)
    lib.call("seg_maxpool2x2_bwd", ptr(dy), ptr(code), ptr(dx), N, H, W, C)
    ub, u = guarded((N, H, W, C), BF16)
    lib.call("seg_maxunpool2x2_fwd", ptr(y), ptr(code), ptr(u), N, H, W, C)
    dub, du = guarded((N, P, Q, C), BF16)
    lib.call("seg_maxunpool2x2_bwd", ptr(dyu), ptr(code), ptr(du), N, H, W, C)
    torch.cuda.synchronize()
    return (y, code, dx, u, du), (yb, cb, dxb, ub, dub)


def run_aten(x, dy, dyu):
    """ATen CUDA on the same bf16 values (NCHW views of the NHWC tensors)."""
    H, W = x.shape[1:3]
    xr = x.permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    y, idx = F.max_pool2d(xr, 2, 2, return_indices=True)
    y.backward(dy.permute(0, 3, 1, 2).contiguous())
    yu = y.detach().clone().requires_grad_(True)
    u = F.max_unpool2d(yu, idx, 2, 2, output_size=(H, W))
    u.backward(dyu.permute(0, 3, 1, 2).contiguous())
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y.detach()), nhwc(idx), nhwc(xr.grad), nhwc(u.detach()), nhwc(yu.grad)


def pool_case(log, N, H, W, C, seed):
    case = f"pool2x2 {N}x{H}x{W}x{C}"
    x = make_pool_input(N, H, W, C, seed)
    g = torch.Generator().manual_seed(seed + 1)
    dy = torch.randn(N, H // 2, W // 2, C, generator=g).bfloat16().to(DEV)
    dyu = torch.randn(N, H, W, C, generator=g).bfloat16().to(DEV)
    ours, guards = run_ours(x, dy, dyu)
    for buf, dt, what in zip(guards, (BF16, U8, BF16, BF16, BF16), ("y", "code", "dx", "unpool y", "unpool dx")):
        check_guard(f"{case} {what}", buf, dt)
    y, code, dx, u, du = ours
    ry, ridx, rdx, ru, rdu = run_aten(x, dy, dyu)
    assert code.max().item() <= 3, f"{case}: a code was not written"
    P, Q = H // 2, W // 2
    p = torch.arange(P, device=DEV).view(1, P, 1, 1)
    q = torch.arange(Q, device=DEV).view(1, 1, Q, 1)
    c = code.long()
    assert torch.equal((2 * p + c // 2) * W + 2 * q + c % 2, ridx), f"{case}: codes differ from ATen's indices"
    assert torch.equal(bits(y), bits(ry)), f"{case}: pooled values differ from ATen's"
    assert torch.equal(bits(dx), bits(rdx)), f"{case}: max-pool gradient differs from ATen's"
    assert torch.equal(bits(u), bits(ru)), f"{case}: unpooled values differ from ATen's"
    assert torch.equal(bits(du), bits(rdu)), f"{case}: max-unpool gradient differs from ATen's"
    again, _ = run_ours(x, dy, dyu)
    for a, b, what in zip(ours, again, ("y", "code", "dx", "unpool y", "unpool dx")):
        assert torch.equal(bits(a), bits(b)), f"{case}: {what} not bit-reproducible"
    nan_in = int(torch.isnan(x.float()).sum())
    log(f"{case}: bit-identical to ATen (values, indices, both gradients); NaN inputs {nan_in}, "
        f"pooled vectors {N * P * Q * C // 8} (grid cap {grid_cap()})")


@pytest.mark.parametrize("C", [8, 64, 512])
@pytest.mark.parametrize("hw", [(2, 2), (3, 3), (2, 7), (3, 8), (16, 16), (17, 23), (50, 75), (25, 37)])
def test_pool_unpool_match_aten(log, hw, C):
    pool_case(log, 2, hw[0], hw[1], C, seed=hw[0] * 131 + hw[1] + C)


@pytest.mark.parametrize("extra", [-1, 0, 1])
def test_pool_unpool_at_the_grid_cap(log, extra):
    """N * P * Q * C / 8 = SMs * 8 * 256 + extra pooled vectors: the last one sits on either side of one full grid pass.
    H is odd, so the scatter kernels (one window row more, the dropped row) cover one more."""
    n = grid_cap() + extra
    pool_case(log, 1, 2 * n + 1, 2, 8, seed=40 + extra)


def test_pool_unpool_several_grid_strides(log):
    n = 3 * grid_cap() + 5
    pool_case(log, 1, 2 * n + 1, 3, 8, seed=45)
    pool_case(log, 2, 2 * (grid_cap() // 64) + 1, 2 * 3 + 1, 64, seed=46)


def test_pool_entry_points_reject_bad_channels():
    x = torch.zeros(1, 4, 4, 12, dtype=BF16, device=DEV)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.maxpool2x2_fwd(x)


# ------------------------------------------------------------------------------------------------ the classifier conv
@pytest.mark.parametrize("N,H,W", [(2, 64, 64), (2, 50, 75), (1, 512, 512)])
def test_classifier_conv_conformance(log, N, H, W):
    """stage5_decoder.6: Conv2d(64, 19, 3, p1) with bias and fp32 NHWC output (dense, as the model writes it); its data
    gradient over a 19-channel dY in a zero-padded pitch-24 buffer (what the head's loss backward hands it) and its weight
    gradient, each element within conv_check's float64 bound, bit-reproducible, with guards intact."""
    K, C = 19, 64
    seed = H + W
    x = cc.make_x(N, H, W, C, seed)
    w = cc.make_w(K, C, 3, 3, seed + 1)
    bias = (torch.randn(K, generator=torch.Generator().manual_seed(seed + 2)) * 0.1).float()
    wp = ops.pack_weight(w.float().to(DEV))
    xd = x.to(DEV, BF16).contiguous()
    case = f"classifier conv {N}x{H}x{W} 64->19"
    r = cc.fprop_ref(x, w, 1, 1, 1, bias=bias)
    outs = []
    for _ in range(2):
        g = cc.Guarded(N, H, W, K, F32, 0, 0, device=DEV)
        ops.conv2d_fwd(xd, wp, K, 3, 3, 1, 1, 1, out=g.view, bias=bias.to(DEV), impl=IMPL_AUTO)
        torch.cuda.synchronize()
        cc.check_guards(case + " fprop", g.buf, g.guard_mask())
        cc.check_written(case + " fprop", g.view)
        outs.append(g.view.clone())
    uf = cc.check_elements(case + " fprop", outs[0], r, False)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), f"{case}: fprop not bit-reproducible"

    dy = cc.make_x(N, H, W, K, seed + 3)
    dbuf = torch.zeros(N, H, W, 24, dtype=BF16, device=DEV)
    dbuf[..., :K] = dy.to(DEV, BF16)
    dyd = dbuf[..., :K]
    r = cc.dgrad_ref(dy, w, (N, H, W, C), 1, 1, 1)
    outs = []
    for _ in range(2):
        g = cc.Guarded(N, H, W, C, BF16, cc.GUARD, cc.GUARD, device=DEV)
        ops.conv2d_dgrad(dyd, wp, (N, H, W, C), 3, 3, 1, 1, 1, out=g.view, impl=IMPL_AUTO)
        torch.cuda.synchronize()
        cc.check_guards(case + " dgrad", g.buf, g.guard_mask())
        cc.check_written(case + " dgrad", g.view)
        outs.append(g.view.clone())
    ud = cc.check_elements(case + " dgrad", outs[0], r, True)
    assert torch.equal(outs[0].view(I16), outs[1].view(I16)), f"{case}: dgrad not bit-reproducible"
    tc = ops.conv2d_dgrad(dyd, wp, (N, H, W, C), 3, 3, 1, 1, 1, impl=IMPL_TC)
    assert torch.equal(tc.view(I16), outs[0].view(I16)), f"{case}: AUTO dgrad did not take the wgmma path"

    r = cc.wgrad_ref(dy, x, 3, 3, 1, 1, 1)
    d = lib.make_conv_desc(N, H, W, C, K, 3, 3, 1, 1, 1, ldx=C, ldy=24)
    nws = int(lib.load().seg_conv2d_wgrad_workspace_floats(ctypes.byref(d), IMPL_AUTO))
    splits = nws // (9 * K * C) if nws else 1
    outs = []
    for _ in range(2):
        f = cc.FlatGuarded((9, K, C), F32, device=DEV)
        f.view.zero_()
        ops.conv2d_wgrad(dyd, xd, 3, 3, 1, 1, 1, out=f.view, impl=IMPL_AUTO)
        torch.cuda.synchronize()
        cc.check_guards(case + " wgrad", f.buf, f.guard_mask())
        outs.append(f.view.clone())
    uw = cc.check_elements(case + " wgrad", outs[0], r, False, splits=splits)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), f"{case}: wgrad not bit-reproducible"
    log(f"{case}: usage fprop={uf:.4f} dgrad={ud:.4f} wgrad={uw:.4f} (splits={splits})")


# ------------------------------------------------------------------------------------------------ the model
def build(nc, seed, **kw):
    sd = osn.segnet_state_dict(nc, seed=seed, randomize_bn=True)
    m = seg_b200.SegNet(nc, pretrained=False, **kw)
    m.load_state_dict(sd, strict=True)
    return sd, m.cuda()


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def cosine(a, b):
    return F.cosine_similarity(a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten(), dim=0).item()


def argmax_report(log, tag, out, ref):
    """Argmax agreement; pixels whose top-2 margin is within twice the max error are undecidable."""
    err = (out.detach().cpu() - ref).abs().max().item()
    top2 = ref.topk(2, dim=1).values
    safe = (top2[:, 0] - top2[:, 1]) > 2 * err
    am_e, am_r = out.detach().argmax(1).cpu(), ref.argmax(1)
    agree_all = (am_e == am_r).float().mean().item()
    agree_safe = (am_e[safe] == am_r[safe]).float().mean().item() if safe.any() else 1.0
    log(f"{tag} argmax vs oracle: all pixels {agree_all:.5f}; decidable pixels ({safe.float().mean().item():.3f} of map) {agree_safe:.5f}")
    return agree_all, agree_safe


def bf16_control(sd, x, y, train):
    """The oracle's forward and backward run by ATen on the GPU in bf16 (cuDNN convs, bf16 pools): the error a plain bf16
    implementation of the same model makes.  Returns (logits fp32 CPU, {name: grad})."""
    bsd = {k: (v.to(DEV, BF16) if v.is_floating_point() else v.to(DEV)) for k, v in sd.items()}
    for k, v in bsd.items():
        if k.endswith(("weight", "bias")):
            v.requires_grad_(True)
    out = osn.segnet_forward(bsd, x.to(DEV, BF16), train=train)
    loss = F.cross_entropy(out.float(), y.to(DEV), ignore_index=255)
    loss.backward()
    return out.detach().float().cpu(), {k: v.grad.float().cpu() for k, v in bsd.items() if v.grad is not None}


BOUND_FACTOR = 4.0  # the engine may be this many times further from the fp32 oracle than the ATen bf16 run is


@pytest.mark.parametrize("hw", [(64, 64), (50, 75)], ids=["64x64", "50x75"])
def test_frozen_bn_train_step_parity(log, hw):
    """Frozen BatchNorm: every forward and backward kernel in context against the fp32 oracle, with the logits bound and
    the gradient-direction bound set from an ATen bf16 run of the same model.  Near-ties inside a pool window can send a
    gradient to another pixel in bf16, so gradients are compared by cosine."""
    sd, m = build(19, 11)
    x, y = synth.make_batch(2, hw[0], hw[1], 19, 255, seed=9051)
    osd = om.clone_sd(sd, requires_grad=True)
    ref = osn.segnet_forward(osd, x, train=False)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    ctrl_out, ctrl_grads = bf16_control(sd, x, y, train=False)
    m.train()
    m.freeze_bn()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[frozen-BN segnet {hw[0]}x{hw[1]}]"
    e, ec = relerr(out, ref), relerr(ctrl_out, ref)
    log(f"{tag} logits rel_err vs fp32 oracle {e:.3e} (ATen bf16 {ec:.3e}); loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert out.shape == ref.shape == (2, 19) + hw and e <= BOUND_FACTOR * ec
    _, agree_safe = argmax_report(log, tag, out, ref.detach())
    assert agree_safe == 1.0
    cos, ccos = {}, {}
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        if osd[name].grad.abs().max() > 0:
            cos[name] = cosine(p.grad, osd[name].grad)
            ccos[name] = cosine(ctrl_grads[name], osd[name].grad)
    worst, cworst = min(cos, key=cos.get), min(ccos, key=ccos.get)
    log(f"{tag} grads vs fp32 oracle: min cosine {cos[worst]:.5f} at {worst} (ATen bf16 {ccos[cworst]:.5f} at {cworst})")
    assert 1 - cos[worst] <= BOUND_FACTOR * (1 - ccos[cworst]), (cos[worst], worst, ccos[cworst], cworst)
    esd = m.state_dict()
    assert all(torch.equal(esd[k].cpu(), sd[k]) for k in esd if "running_" in k)


def test_eval_forward_and_batchstat_train_step(log):
    sd, m = build(19, 12)
    x, y = synth.make_batch(2, 50, 75, 19, 255, seed=9052)
    osd = om.clone_sd(sd, requires_grad=True)
    m.eval()
    with torch.no_grad():
        ev = m(x.cuda())
        ev_ref = osn.segnet_forward(osd, x, train=False)
    ctrl, _ = bf16_control(sd, x, y, train=False)
    log(f"[eval segnet] logits rel_err vs fp32 oracle {relerr(ev, ev_ref):.3e} (ATen bf16 {relerr(ctrl, ev_ref):.3e})")
    assert ev.shape == ev_ref.shape and relerr(ev, ev_ref) <= BOUND_FACTOR * relerr(ctrl, ev_ref)
    ref = osn.segnet_forward(osd, x, train=True)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    m.train()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    log(f"[batch-stat segnet] logits rel_err {relerr(out, ref):.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert abs(loss.item() - ref_loss.item()) < 0.05 * abs(ref_loss.item())
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
    esd = m.state_dict()
    for k in ("stage1_encoder.1.running_mean", "stage1_encoder.1.running_var"):
        assert relerr(esd[k], osd[k]) < 1e-2, k
    assert all(int(esd[k]) == 1 for k in esd if k.endswith("num_batches_tracked"))


def _model(seed, nc=7):
    m = seg_b200.SegNet(nc, pretrained=False)
    m.load_state_dict(osn.segnet_state_dict(nc, seed=seed, randomize_bn=True), strict=True)
    return m.cuda().train()


def _crit(name, C):
    if name == "ce":
        return losses.CrossEntropyLoss2d(ignore_index=255)
    if name == "wce":
        return losses.CrossEntropyLoss2d(weight=lc.weights(C, 5).cuda(), ignore_index=255)
    return losses.FocalLoss(ignore_index=255)


@pytest.mark.parametrize("name", ["ce", "wce", "focal"])
@pytest.mark.parametrize("hw", [(64, 64), (50, 75)], ids=["64x64", "50x75"])
def test_fused_step_first_loss_and_counters_equal_plugin(log, name, hw):
    x, y = synth.make_batch(2, hw[0], hw[1], 7, 255, seed=9053)
    xd, yd = x.cuda(), y.cuda()
    crit = _crit(name, 7)
    with torch.no_grad():
        out = _model(41)(xd)
        ref = float(crit(out, yd))
        want = ops.eval_metrics_nchw(out, yd, 7)
    s = FusedTrainStep(_model(41), lr=0.005, loss=crit, metrics=True)
    got = float(s.step(xd, yd))
    log(f"fused step [segnet {name} {hw[0]}x{hw[1]}] first loss {got:.7f}, plugin {ref:.7f}")
    assert abs(got - ref) <= 1e-5 * abs(ref)
    assert torch.equal(s.seg_counters, want)


def test_fused_step_graph_replay_is_bit_identical():
    x, y = synth.make_batch(2, 50, 75, 7, 255, seed=9054)
    xd, yd = x.cuda(), y.cuda()
    se = FusedTrainStep(_model(42), lr=0.005, metrics=True)
    sg = FusedTrainStep(_model(42), lr=0.005, metrics=True, cuda_graph=True)
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
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9055)
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
    """model.cuda_graphs(): the replayed plugin step gives the eager step's output and gradients bit for bit."""
    x, y = synth.make_batch(2, 50, 75, 7, 255, seed=9056)
    xd, yd = x.cuda(), y.cuda()
    m = _model(45).cuda_graphs(True, warmup=1)
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    res = []
    for _ in range(4):  # eager (warm-up), capture, replay, replay
        for p in m.parameters():
            p.grad = None
        out = m(xd)
        loss = crit(out, yd)
        loss.backward()
        res.append((out.detach().clone(), loss.detach().clone(), [p.grad.clone() for p in m.parameters()]))
    assert m._graph_entries, "no graph was captured"
    for o, l, g in res[1:]:
        assert torch.equal(o, res[0][0]) and torch.equal(l, res[0][1])
        assert all(torch.equal(a, b) for a, b in zip(g, res[0][2]))
    m.cuda_graphs(False)


def test_small_input_raises_before_any_launch():
    m = _model(47)
    n = lib.launch_count()
    with pytest.raises(ValueError, match="31x64"):
        m(torch.zeros(1, 3, 31, 64, device=DEV))
    assert lib.launch_count() == n


@pytest.mark.parametrize("size", [512, 513])
def test_full_size_graph_step(log, size):
    """One 8 x 3 x size^2 fused graph step (the configs' crop and batch; 513 drops a row and a column at the first pool) has
    a finite loss."""
    x, y = synth.make_batch(8, size, size, 19, 255, seed=9058)
    s = FusedTrainStep(_model(46, nc=19), lr=0.01, cuda_graph=True)
    losses_ = [float(s.step(x.cuda(), y.cuda())) for _ in range(2)]
    torch.cuda.synchronize()
    log(f"[segnet 8x3x{size}x{size} graph step] losses {losses_[0]:.6f} {losses_[1]:.6f}")
    assert all(v == v and abs(v) < 1e3 for v in losses_)
    s.release_graph()
