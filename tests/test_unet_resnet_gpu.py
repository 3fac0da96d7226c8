"""UNetResnet on the H100: the transposed convolutions (the wgmma dgrad / fprop / wgrad of the mirrored conv) against the
float64 F.conv_transpose2d with tests/conv_check.py's per-element bound, the full-resolution head (logits transposes bit for
bit, the fused loss seg_nhwc_loss_* against tests/loss_check.py's float64 references and eval_metrics), the model against the
fp32 oracle of oracle/unet_resnet.py (pinned to the reference by tests/golden/unet_resnet.npz), and FusedTrainStep and the
plugin surface on the model."""
import ctypes
import os
import time

import pytest
import torch
import torch.nn.functional as F

import conv_check as cc
import loss_check as lc
from oracle import losses as ol
from oracle import models as om
from oracle import synth
from oracle import unet_resnet as ou

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import lib, losses, ops
    from seg_b200.engine import Act, FullResHead
    from seg_b200.lib import IMPL_AUTO, IMPL_SIMT, IMPL_TC, ptr
    from seg_b200.train import FusedTrainStep
else:  # keep collection working without a GPU
    IMPL_AUTO, IMPL_SIMT, IMPL_TC = 0, 1, 2

DEV = "cuda"
F32, F64, I64, I32, BF16 = torch.float32, torch.float64, torch.int64, torch.int32, torch.bfloat16
KIND = {"ce": 0, "wce": 1, "focal": 2}


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "unet_resnet.txt"), "a")

    def write(line):
        print(line)
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def place(t, lead=8):
    """bf16 NHWC device tensor holding t as a channel slice at offset `lead` of a sentinel-filled buffer whose pitch is a
    multiple of 8 (a kernel reading outside the slice produces NaNs)."""
    N, H, W, C = t.shape
    trail = cc.GUARD + (-(lead + C + cc.GUARD)) % 8
    buf = cc.sentinel_fill(torch.empty(N, H, W, lead + C + trail, dtype=BF16, device=DEV))
    buf[..., lead:lead + C] = t.to(DEV, BF16)
    return buf[..., lead:lead + C]


def guarded(N, H, W, C, old=None):
    """A sentinel-guarded concat slice (8 guard channels before it, a pitch that is a multiple of 8) holding `old` or the
    sentinel."""
    g = cc.Guarded(N, H, W, C, BF16, cc.GUARD, cc.GUARD + (-(cc.GUARD + C + cc.GUARD)) % 8, device=DEV)
    if old is not None:
        g.view.copy_(old.to(DEV, BF16))
    return g


# ------------------------------------------------------------------------------------------------ transposed conv
DECODER_SHAPES = [(192, 128), (128, 96), (96, 64), (64, 48), (48, 32)]  # upconv1..5 (Cin -> Cout), unet.py:147-160
SIZES = {"h1": (1, 1), "odd": (5, 7), "even": (6, 4)}


def _convt64(x, w):
    """float64 F.conv_transpose2d(k=4, s=2, p=1) of NHWC x [N,h,w,Cin] with weight [Cin,Cout,4,4]; NHWC result."""
    return cc.nhwc(F.conv_transpose2d(cc.nchw(x.double()), w.double(), None, 2, 1))


def _three_runs(fn, out_view_factory):
    """fn(out, impl) twice on the wgmma path and once under AUTO; returns the outputs (the guards are checked by the caller)."""
    res = []
    for impl in (IMPL_TC, IMPL_TC, IMPL_AUTO):
        g = out_view_factory()
        fn(g.view, impl)
        torch.cuda.synchronize()
        res.append(g)
    return res


@pytest.mark.parametrize("beta", [0.0, 1.0], ids=["beta0", "beta1"])
@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("cin,cout", DECODER_SHAPES, ids=[f"{a}to{b}" for a, b in DECODER_SHAPES])
def test_conv_transpose_conformance(log, cin, cout, size, beta):
    """ConvTranspose2d(cin, cout, 4, 2, 1): forward (= dgrad of the mirrored conv into a concat slice), data gradient (= its
    fprop over dY) and weight gradient (= its wgrad with the operands swapped), each checked element by element against the
    float64 F.conv_transpose2d and its autograd of the bf16 operands, with guards unchanged and two wgmma runs bit-identical.
    AUTO must give the wgmma result bit for bit (the CUDA-core kernel sums in another order, which the case asserts too)."""
    N = 2
    h, w = SIZES[size]
    Ho, Wo = 2 * h, 2 * w
    seed = cin + 7 * h + int(beta)
    x = cc.make_x(N, h, w, cin, seed)
    W = cc.make_w(cin, cout, 4, 4, seed + 1)       # [Cin, Cout, 4, 4] = the OIHW weight of the Conv2d(Cout -> Cin)
    dY = cc.make_x(N, Ho, Wo, cout, seed + 2)
    wp = ops.pack_weight(W.float().to(DEV))
    case = f"convT {cin}->{cout} {N}x{h}x{w} beta={beta:g}"

    # forward
    old = cc.make_x(N, Ho, Wo, cout, seed + 3) if beta else None
    r = cc.dgrad_ref(x, W, (N, Ho, Wo, cout), 2, 1, 1, beta=beta, old=old)
    assert torch.allclose(r.staged, _convt64(x, W), rtol=1e-12, atol=1e-300)
    xin = place(x)
    runs = _three_runs(lambda out, impl: ops.conv2d_dgrad(xin, wp, (N, Ho, Wo, cout), 4, 4, 2, 1, 1, out=out, beta=beta, impl=impl),
                       lambda: guarded(N, Ho, Wo, cout, old))
    for g in runs:
        cc.check_guards(case + " fwd", g.buf, g.guard_mask())
        cc.check_written(case + " fwd", g.view)
    u_f = cc.check_elements(case + " fwd", runs[0].view, r, True, staged=beta != 0.0)
    assert torch.equal(runs[0].view.view(torch.int16), runs[1].view.view(torch.int16)), f"{case}: fwd not bit-reproducible"
    assert torch.equal(runs[0].view.view(torch.int16), runs[2].view.view(torch.int16)), f"{case}: AUTO did not take the wgmma path"

    # data gradient: dX = conv2d(dY, W) (the autograd of F.conv_transpose2d w.r.t. its input)
    old = cc.make_x(N, h, w, cin, seed + 4) if beta else None
    r = cc.fprop_ref(dY, W, 2, 1, 1, beta=beta, old=old)
    xr = cc.nchw(x.double()).clone().requires_grad_(True)
    F.conv_transpose2d(xr, W.double(), None, 2, 1).backward(cc.nchw(dY.double()))
    assert torch.allclose(r.staged, cc.nhwc(xr.grad), rtol=1e-12, atol=1e-300)
    dyin = place(dY)
    runs = _three_runs(lambda out, impl: ops.conv2d_fwd(dyin, wp, cin, 4, 4, 2, 1, 1, out=out, beta=beta, impl=impl),
                       lambda: guarded(N, h, w, cin, old))
    for g in runs:
        cc.check_guards(case + " dgrad", g.buf, g.guard_mask())
        cc.check_written(case + " dgrad", g.view)
    u_d = cc.check_elements(case + " dgrad", runs[0].view, r, True, staged=beta != 0.0)
    assert torch.equal(runs[0].view.view(torch.int16), runs[1].view.view(torch.int16)), f"{case}: dgrad not bit-reproducible"
    assert torch.equal(runs[0].view.view(torch.int16), runs[2].view.view(torch.int16)), f"{case}: AUTO did not take the wgmma path"

    # weight gradient: packed [16][Cin][Cout], accumulated onto dw_old (unpack_wgrad turns it into [Cin, Cout, 4, 4])
    dw_old = torch.randn(16, cin, cout, generator=torch.Generator().manual_seed(seed + 5)).double()
    r = cc.wgrad_ref(x, dY, 4, 4, 2, 1, 1, old=dw_old)
    Wr = W.double().clone().requires_grad_(True)
    F.conv_transpose2d(cc.nchw(x.double()), Wr, None, 2, 1).backward(cc.nchw(dY.double()))
    assert torch.allclose(r.staged, cc.pack_w(Wr.grad), rtol=1e-12, atol=1e-300)
    d = lib.make_conv_desc(N, Ho, Wo, cout, cin, 4, 4, 2, 1, 1, ldx=ops.ld(dyin), ldy=ops.ld(xin))
    outs = {}
    for run, impl in enumerate((IMPL_TC, IMPL_TC, IMPL_AUTO, IMPL_SIMT)):
        nws = int(lib.load().seg_conv2d_wgrad_workspace_floats(ctypes.byref(d), impl))
        splits = nws // (16 * cin * cout) if nws else 1
        f = cc.FlatGuarded((16, cin, cout), F32, device=DEV)
        f.view.copy_(dw_old.float())
        ws = torch.full((nws,), float("nan"), device=DEV) if nws else None
        lib.call("seg_conv2d_wgrad", ctypes.byref(d), ptr(xin), ptr(dyin), ptr(f.view), ptr(ws), impl)
        torch.cuda.synchronize()
        cc.check_guards(case + " wgrad", f.buf, f.guard_mask())
        outs[run] = (f.view.clone(), splits)
    u_w = cc.check_elements(case + " wgrad", outs[0][0], r, False, splits=outs[0][1])
    cc.check_elements(case + " wgrad simt", outs[3][0], r, False)
    assert torch.equal(outs[0][0].view(torch.int32), outs[1][0].view(torch.int32)), f"{case}: wgrad not bit-reproducible"
    assert torch.equal(outs[0][0].view(torch.int32), outs[2][0].view(torch.int32)), f"{case}: AUTO did not take the wgmma path"
    got = ops.unpack_wgrad(outs[0][0], (cin, cout, 4, 4))
    assert torch.equal(got.cpu(), outs[0][0].cpu().reshape(4, 4, cin, cout).permute(2, 3, 0, 1))
    log(f"{case}: usage fwd={u_f:.4f} dgrad={u_d:.4f} wgrad={u_w:.4f} (splits={outs[0][1]})")


def test_auto_and_simt_differ_on_a_decoder_shape():
    """The AUTO == wgmma assertions above are only informative when the CUDA-core kernel would give other bits."""
    x = cc.make_x(2, 6, 4, 192, 1)
    W = cc.make_w(192, 128, 4, 4, 2)
    wp = ops.pack_weight(W.float().to(DEV))
    xin = place(x)
    a = ops.conv2d_dgrad(xin, wp, (2, 12, 8, 128), 4, 4, 2, 1, 1, impl=IMPL_AUTO)
    s = ops.conv2d_dgrad(xin, wp, (2, 12, 8, 128), 4, 4, 2, 1, 1, impl=IMPL_SIMT)
    assert not torch.equal(a.view(torch.int16), s.view(torch.int16))


def test_tape_conv_transpose_matches_the_kernels():
    """Tape.conv_transpose under the model's AUTO setting issues exactly the wgmma calls checked above, forward and backward,
    and accumulates into an existing input gradient."""
    from seg_b200.engine import ConvSpec, Tape
    torch.manual_seed(3)
    mod = torch.nn.ConvTranspose2d(64, 48, 4, 2, 1, bias=False).cuda()
    spec = ConvSpec("up", mod)
    x = torch.randn(2, 5, 7, 64, device=DEV).bfloat16()
    tape = Tape(True)
    xa = Act(x)
    y = tape.conv_transpose(xa, spec)
    assert y.t.shape == (2, 10, 14, 48)
    wp = ops.pack_weight(mod.weight.detach())
    assert torch.equal(y.t, ops.conv2d_dgrad(x, wp, (2, 10, 14, 48), 4, 4, 2, 1, 1, impl=IMPL_TC))
    dy = torch.randn(2, 10, 14, 48, device=DEV).bfloat16()
    prev = torch.randn(2, 5, 7, 64, device=DEV).bfloat16()
    xa.grad, xa._written = prev.clone(), True
    y.grad = dy
    tape.backward()
    assert torch.equal(xa.grad, ops.conv2d_fwd(dy, wp, 64, 4, 4, 2, 1, 1, out=prev.clone(), beta=1.0, impl=IMPL_TC))
    want = ops.unpack_wgrad(ops.conv2d_wgrad(x, dy, 4, 4, 2, 1, 1, impl=IMPL_TC), (64, 48, 4, 4))
    assert torch.equal(tape.grads[mod.weight], want)


# ------------------------------------------------------------------------------------------------ full-resolution head
def test_logits_transposes_are_exact():
    g = torch.Generator().manual_seed(5)
    N, H, W, C = 2, 9, 13, 19
    buf = torch.randn(N, H, W, C + 5, generator=g).to(DEV)
    x = buf[..., 2:2 + C]  # conv7 writes a dense [N,H,W,C]; a pitch is accepted too
    head = FullResHead(Act(x))
    y = head.logits()
    assert torch.equal(y.cpu(), x.cpu().permute(0, 3, 1, 2))
    dy = torch.randn(N, C, H, W, generator=g)
    head.logits_bwd(dy.to(DEV))
    dx = head.act.grad
    assert ops.ld(dx) == 24 and dx.shape == (N, H, W, C)
    assert torch.equal(dx.cpu(), dy.permute(0, 2, 3, 1).bfloat16())
    full = dx.as_strided((N, H, W, 24), dx.stride())
    assert (full[..., C:] == 0).all()


def run_nhwc_loss(log, case, z, C, t, kind="ce", gamma=0.0, mean=True, weight=None, gscale=0.75, ignore=255):
    """z: fp32 NHWC logits [N, H, W, C], placed as a channel slice (8 sentinel lanes on each side) of a wider pitch."""
    t0 = time.time()
    N, H, W, _ = z.shape
    buf = cc.sentinel_fill(torch.empty(N, H, W, 8 + C + 8, dtype=F32, device=DEV))
    buf[..., 8:8 + C] = z.to(DEV)
    zd, ld = buf[..., 8:8 + C], 8 + C + 8
    td = t.to(DEV)
    wd = None if weight is None else weight.to(DEV, F32).contiguous()
    gs = torch.tensor([gscale], dtype=F32, device=DEV)
    lddx = C + 5
    M = N * H * W
    blocks, iters, capped = lc.nchw_grid(M, sms())
    runs = []
    for _ in range(2):
        accum = torch.zeros(2, dtype=F64, device=DEV)
        cbuf = lc.int_sentinel_fill(torch.empty(8 + 2 + 3 * C + 8, dtype=I64, device=DEV))
        cnt = cbuf[8:8 + 2 + 3 * C]
        cnt.zero_()
        lib.call("seg_nhwc_loss_fwd", ptr(zd), ld, ptr(td), N, H, W, C, int(ignore), ptr(wd), KIND[kind], float(gamma), ptr(accum),
                 ptr(cnt))
        loss = torch.empty(1, dtype=F32, device=DEV)
        lib.call("seg_loss_finalize", ptr(accum), int(mean), ptr(loss))
        dx = cc.FlatGuarded((M, lddx), BF16, device=DEV)
        lib.call("seg_nhwc_loss_bwd", ptr(zd), ld, ptr(td), N, H, W, C, int(ignore), ptr(wd), KIND[kind], float(gamma), int(mean),
                 ptr(accum), ptr(gs), ptr(dx.view), lddx)
        torch.cuda.synchronize()
        cc.check_guards(case, dx.buf, dx.guard_mask())
        cc.check_written(case, dx.view)
        lc.check_int_guards(case + " counters", cbuf, 8, 2 + 3 * C)
        runs.append((accum.clone(), loss.clone(), dx.view.clone(), cnt.clone()))
    a, b = runs
    assert torch.equal(a[0][1:], b[0][1:]) and torch.equal(a[1].view(I32), b[1].view(I32)), f"{case}: loss not bit-reproducible"
    assert torch.equal(a[2].view(torch.int16), b[2].view(torch.int16)), f"{case}: dx not bit-reproducible"
    assert torch.equal(a[3], b[3]), f"{case}: counters not bit-reproducible"
    accum, loss, dx, cnt = a
    ref = lc.ShuffleRef(zd.double(), 1, C, td, ignore, kind, wd, gamma, mean)  # the r = 1 shuffle is the NHWC view
    ua = max(ref.loss.check_accum(case, accum), ref.loss.check_accum(case, b[0]))
    ul = ref.loss.check_loss(case, loss.item())
    b = ref.dx_bound(gscale)
    # lc.logits spans 2^-9 .. 2^6 per pixel, so some probabilities (and their gradients) fall below 2^-126, where bf16 is
    # subnormal with a spacing of 2^-133: the relative rounding allowance gets half that spacing added
    b.rnd = b.rnd + 2.0 ** -134
    ug = lc.check(case, "dx", dx[:, :C].reshape(N, H, W, C), b)
    lc.check_pad(case, dx, C)
    lc.check_exact(case, "counters vs eval_metrics", cnt, ops.eval_metrics_nchw(zd.permute(0, 3, 1, 2).contiguous(), td, C).cpu(),
                   ("i",))
    lc.check_exact(case, "counters vs first max", cnt.cpu(), lc.metrics_ref(ref.loss.sm.z, td, C), ("i",))
    log(f"{case}: usage accum0={ua:.4f} loss={ul:.4f} dx={ug:.4f} blocks={blocks} iters={iters} capped={capped} "
        f"time={time.time() - t0:.2f}s")


def nhwc_logits(N, H, W, C, seed, ties_every=0):
    z = lc.logits(N, C, H, W, seed).permute(0, 2, 3, 1).contiguous()
    if ties_every:  # classes 1 and C - 2 equal and maximal at every ties_every-th pixel
        sel = z.view(-1, C)[::ties_every]
        sel[:, 1] = sel.amax(1) + 1
        sel[:, C - 2] = sel[:, 1]
    return z


# (kind, gamma, mean, weighted)
LOSS_KINDS = [("ce", 0.0, True, False), ("wce", 0.0, True, True), ("wce", 0.0, False, True), ("focal", 0.0, True, False),
              ("focal", 0.5, True, True), ("focal", 2.0, True, False), ("focal", 2.0, False, True)]


@pytest.mark.parametrize("C,ignore", [(2, 255), (19, 255), (21, -1), (150, 0)])
def test_nhwc_loss_conformance(log, C, ignore):
    for kind, gamma, mean, weighted in LOSS_KINDS:
        z = nhwc_logits(2, 17, 23, C, 70 + C, ties_every=3 if C > 2 else 0)
        t = lc.labels(2, 17, 23, C, 71 + C, ignore=ignore)
        w = lc.weights(C, 72 + C) if weighted else None  # every fifth class weight is zero
        run_nhwc_loss(log, f"nhwc C={C} ignore={ignore} {kind} g={gamma} mean={mean}", z, C, t, kind, gamma, mean, w, ignore=ignore)
    t = torch.full((2, 17, 23), ignore, dtype=torch.int64)
    for kind, gamma, mean, weighted in LOSS_KINDS:
        w = lc.weights(C, 72 + C) if weighted else None
        run_nhwc_loss(log, f"nhwc C={C} all ignored {kind} g={gamma} mean={mean}", nhwc_logits(2, 17, 23, C, 73), C, t, kind, gamma,
                      mean, w, ignore=ignore)


def test_nhwc_loss_grid_capped(log):
    N, H, W = 2, 400, 401
    assert lc.nchw_grid(N * H * W, sms())[2]
    run_nhwc_loss(log, f"nhwc {N}x{H}x{W} C=19 (grid-capped)", nhwc_logits(N, H, W, 19, 80, ties_every=7), 19, lc.labels(N, H, W, 19, 81))
    run_nhwc_loss(log, f"nhwc {N}x{H}x{W} C=19 focal (grid-capped)", nhwc_logits(N, H, W, 19, 82), 19, lc.labels(N, H, W, 19, 83),
                  "focal", 2.0, True, lc.weights(19, 84))


def test_nhwc_loss_rejects_a_target_of_another_size():
    z = torch.zeros(1, 16, 16, 7, dtype=F32, device=DEV)
    with pytest.raises(ValueError, match=r"\(15, 16\).*\(16, 16\)"):
        ops.nhwc_loss_fwd(z, torch.zeros(1, 15, 16, dtype=torch.int64, device=DEV), 255)


# ------------------------------------------------------------------------------------------------ model vs oracle
def build(nc, seed, **kw):
    sd = ou.unet_resnet_state_dict(nc, seed=seed, randomize_bn=True)
    m = seg_b200.UNetResnet(nc, pretrained=False, **kw)
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


@pytest.mark.parametrize("size", [64, 65])
def test_frozen_bn_train_step_parity(log, size):
    """Frozen BatchNorm: every forward and backward kernel in context (transposed convs into concat slices or through the
    resample, skips written by the trunk into the concats, the full-resolution head) against the fp32 oracle at the bf16
    noise floor."""
    sd, m = build(19, 11)
    x, y = synth.make_batch(2, size, size, 19, 255, seed=9041)
    osd = om.clone_sd(sd, requires_grad=True)
    ref = ou.unet_resnet_forward(osd, x, train=False)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    m.train()
    m.freeze_bn()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[frozen-BN unet_resnet {size}x{size}]"
    e = relerr(out, ref)
    log(f"{tag} logits rel_err vs fp32 oracle {e:.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert out.shape == ref.shape == (2, 19, size, size) and e < 5e-2
    assert abs(loss.item() - ref_loss.item()) < 1e-2 * abs(ref_loss.item())
    _, agree_safe = argmax_report(log, tag, out, ref.detach())
    assert agree_safe == 1.0
    cos = {}
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        if osd[name].grad.abs().max() > 0:
            cos[name] = cosine(p.grad, osd[name].grad)
    worst = min(cos, key=cos.get)
    log(f"{tag} grads vs fp32 oracle: min cosine {cos[worst]:.5f} at {worst}; " +
        " ".join(f"{n}={cos[n]:.5f}" for n in ("upconv1.weight", "upconv3.weight", "upconv5.weight", "conv3.bias", "conv7.weight",
                                               "layer1.2.conv3.weight", "initial.0.0.weight")))
    assert cos[worst] > 0.9, (cos[worst], worst)
    esd = m.state_dict()
    assert all(torch.equal(esd[k].cpu(), sd[k]) for k in esd if "running_" in k)


def test_eval_forward_and_batchstat_train_step(log):
    sd, m = build(19, 12)
    x, y = synth.make_batch(2, 64, 64, 19, 255, seed=9042)
    osd = om.clone_sd(sd, requires_grad=True)
    m.eval()
    with torch.no_grad():
        ev = m(x.cuda())
        ev_ref = ou.unet_resnet_forward(osd, x, train=False)
    log(f"[eval unet_resnet] logits rel_err vs fp32 oracle {relerr(ev, ev_ref):.3e}")
    assert ev.shape == ev_ref.shape and relerr(ev, ev_ref) < 5e-2
    ref = ou.unet_resnet_forward(osd, x, train=True)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    m.train()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    log(f"[batch-stat unet_resnet] logits rel_err {relerr(out, ref):.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert abs(loss.item() - ref_loss.item()) < 0.05 * abs(ref_loss.item())
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
    esd = m.state_dict()
    for k in ("initial.0.1.running_mean", "initial.0.1.running_var"):
        assert relerr(esd[k], osd[k]) < 1e-2, k
    assert all(int(esd[k]) == 1 for k in esd if k.endswith("num_batches_tracked"))


# ------------------------------------------------------------------------------------------------ FusedTrainStep
def _model(seed, nc=7):
    m = seg_b200.UNetResnet(nc, pretrained=False)
    m.load_state_dict(ou.unet_resnet_state_dict(nc, seed=seed, randomize_bn=True), strict=True)
    return m.cuda().train()


def _crit(name, C):
    if name == "ce":
        return losses.CrossEntropyLoss2d(ignore_index=255)
    if name == "wce":
        return losses.CrossEntropyLoss2d(weight=lc.weights(C, 5).cuda(), ignore_index=255)
    return losses.FocalLoss(ignore_index=255)


@pytest.mark.parametrize("name", ["ce", "wce", "focal"])
@pytest.mark.parametrize("size", [64, 65])
def test_fused_step_first_loss_and_counters_equal_plugin(log, name, size):
    x, y = synth.make_batch(2, size, size, 7, 255, seed=9043)
    xd, yd = x.cuda(), y.cuda()
    crit = _crit(name, 7)
    with torch.no_grad():
        out = _model(41)(xd)
        ref = float(crit(out, yd))
        want = ops.eval_metrics_nchw(out, yd, 7)
    s = FusedTrainStep(_model(41), lr=0.005, loss=crit, metrics=True)
    got = float(s.step(xd, yd))
    log(f"fused step [unet_resnet {name} {size}x{size}] first loss {got:.7f}, plugin {ref:.7f}")
    assert abs(got - ref) <= 1e-5 * abs(ref)
    assert torch.equal(s.seg_counters, want)


def test_fused_step_graph_replay_is_bit_identical():
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9044)
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
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9045)
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


def test_fused_step_rejects_a_target_of_another_size():
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9046)
    s = FusedTrainStep(_model(44), lr=0.005)
    for call in (s.step, s.evaluate):
        with pytest.raises(ValueError, match=r"\(60, 64\).*\(64, 64\)"):
            call(x.cuda(), y[:, :60].contiguous().cuda())


def test_plugin_surface_graphs_and_losses():
    """model.cuda_graphs(): the replayed plugin step gives the eager step's output and gradients bit for bit (parameters do not
    move; batch statistics make the output independent of the running statistics).  Dice, CE + Dice and Lovasz run on the
    output and back-propagate."""
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9047)
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
    y[y == 255] = 0
    for crit in (losses.DiceLoss(), losses.CE_DiceLoss(), losses.LovaszSoftmax()):
        for p in m.parameters():
            p.grad = None
        loss = crit(m(xd), y.cuda())
        loss.backward()
        assert torch.isfinite(loss) and all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())


@pytest.mark.parametrize("size", [512, 513])
def test_full_size_graph_step(log, size):
    """One 8 x 3 x size^2 fused graph step (the configs' crop and batch; 513 takes every resample path) has a finite loss."""
    x, y = synth.make_batch(8, size, size, 19, 255, seed=9048)
    s = FusedTrainStep(_model(46, nc=19), lr=0.01, cuda_graph=True)
    losses_ = [float(s.step(x.cuda(), y.cuda())) for _ in range(2)]
    torch.cuda.synchronize()
    log(f"[unet_resnet 8x3x{size}x{size} graph step] losses {losses_[0]:.6f} {losses_[1]:.6f}")
    assert all(v == v and abs(v) < 1e3 for v in losses_)
    s.release_graph()
