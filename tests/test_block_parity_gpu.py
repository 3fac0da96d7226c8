"""Teacher-forced per-block parity at the real C3 / C2 shapes, in batch-statistics TRAIN mode (VERDICT r1, item 1b).

Whole-model comparisons of a ~100-layer BatchNorm network mix every layer's rounding; here every block is checked on its
own, in context-free isolation: the fp32 CPU oracle runs the full network once at the BASELINE size (batch 4, 513x513 for
DeepLabV3+/ResNet-101; 473x473 for PSPNet/ResNet-50, reference initialisers) and records every block's input and the
gradient arriving at its output.  Each block is then fed, on BOTH sides, the same bf16-rounded input and the same
bf16-rounded upstream gradient:

    oracle : fp32 ATen, the reference's arithmetic (torchvision Bottleneck / models/resnet.py:100-121,
             deeplabv3_plus.py:286-297 ASSP, :323-330 Decoder, pspnet.py:31-38 _PSPModule + classifier)
    engine : the same block through seg_b200's tape — wgmma fprop/dgrad/wgrad, BN statistics in the conv epilogue,
             bn_apply, bn_bwd_reduce / bn_bwd_apply, bilinear, adaptive pool, concat-free buffers — at exactly the shapes
             bench.py launches (M = 4*129^2, 4*65^2, 4*33^2; persistent tiles, one-wave split-K)

Next to every engine number stands the CONTROL: the same oracle block run by ATen in bf16 (torch.autocast on the GPU) on the
same inputs — the noise floor of bf16 storage.  Asserted per block: forward max-norm relative error <= 1e-2; relative L2
error of the input gradient, of every weight gradient and of every BN gamma / beta gradient <= 2e-2; or <= 1.5 x the
control where bf16 itself cannot do better (the image-pooling BatchNorm over 4 samples in ASPP / PSP bin 1; ReLU-mask
flips in every gradient).  Chaos cannot hide here: a block is 3-10 kernels deep.
"""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import losses as ol
from oracle import models as om
from oracle import synth, weights

if torch.cuda.is_available():
    import seg_b200
    from seg_b200.engine import Act

FWD_TOL, DGRAD_TOL, PGRAD_TOL = 1e-2, 2e-2, 2e-2


def log(gpu_out_dir, msg):
    print(msg)
    with open(os.path.join(gpu_out_dir, "parity_blocks.txt"), "a") as f:
        f.write(msg + "\n")


def bf(t):
    return t.detach().to(torch.bfloat16).float()


def relmax(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def nhwc(t):
    return t.detach().permute(0, 2, 3, 1).contiguous().to("cuda", torch.bfloat16)


def nchw(t):
    return t.detach().float().permute(0, 3, 1, 2).cpu()


def out_grad_nhwc(g_nchw, C):
    """Upstream gradient as the engine holds it: NHWC bf16 with the channel pitch padded to a multiple of 8."""
    ld = (C + 7) // 8 * 8
    buf = torch.zeros(g_nchw.shape[0], g_nchw.shape[2], g_nchw.shape[3], ld, dtype=torch.bfloat16, device="cuda")
    buf[..., :C] = g_nchw.detach().permute(0, 2, 3, 1).to("cuda", torch.bfloat16)
    return buf[..., :C]


class Recorder:
    """(name, fn(sd, *inputs) -> output, inputs, output) of every block the oracle ran (see `_run`)."""

    def __init__(self):
        self.steps = []


def rell2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def oracle_block(fn, sd, xs, g, device, autocast):
    """fn on `device`; autocast=True is the ATen-bf16 CONTROL (cuDNN bf16 convolutions, bf16 activations)."""
    osd = om.clone_sd({k: v.to(device) for k, v in sd.items()}, requires_grad=True)
    xin = [t.to(device).clone().requires_grad_(True) for t in xs]
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        out = fn(osd, *xin)
    out.backward(g.to(device).to(out.dtype))
    return out.detach().float().cpu(), [t.grad.detach().float().cpu() for t in xin], osd


def check_block(gpu_out_dir, tag, fn, in_tensors, g_out, engine_fn, m, prefixes, sd):
    """fn(osd, *inputs) = oracle block; engine_fn(tape, *acts) = engine block.  in_tensors: oracle NCHW fp32 inputs,
    g_out: gradient at the block output.  prefixes: state_dict prefixes of the block's parameters.

    Metrics against the fp32 oracle on the SAME bf16-rounded inputs: max-norm relative error for the forward; relative L2
    error for every gradient.  (Max-norm is meaningless for the gradient of a ReLU network in reduced precision: an
    activation within one bf16 ulp of zero flips its mask and moves that element's gradient by its full magnitude —
    measured below on ATen's own bf16 path, the CONTROL, which shows the same 0.1-0.5 max-norm figures.)  The engine must
    be within 1e-2 (forward) / 2e-2 (gradients), or within 1.5x the control where bf16 itself cannot do better."""
    xs = [bf(t) for t in in_tensors]
    g = bf(g_out)
    bsd = {k: v for k, v in sd.items() if any(k.startswith(p) for p in prefixes)}
    ref_out, ref_dx, osd = oracle_block(fn, bsd, xs, g, "cpu", False)
    ctl_out, ctl_dx, csd = oracle_block(fn, bsd, xs, g, "cuda", True)
    # ---- engine on the same inputs ----
    m.train()
    tape = m._new_tape(True, True)
    acts = [Act(nhwc(t)) for t in xs]
    out = engine_fn(tape, *acts)
    C = out.t.shape[-1]
    out.grad = out_grad_nhwc(g, C) if out.t.dtype == torch.float32 else nhwc(g)
    tape.backward()
    torch.cuda.synchronize()
    res = {"fwd(max)": (relmax(nchw(out.t), ref_out), relmax(ctl_out, ref_out)),
           "fwd(l2)": (rell2(nchw(out.t), ref_out), rell2(ctl_out, ref_out))}
    for i, a in enumerate(acts):
        res[f"dx{i}(l2)"] = (rell2(nchw(a.grad), ref_dx[i]), rell2(ctl_dx[i], ref_dx[i]))
    names = [k for k in om.param_names(osd) if osd[k].grad is not None]
    params = dict(m.named_parameters())
    worst = {"wgrad(l2)": (0.0, 0.0, None), "bn/bias grad(l2)": (0.0, 0.0, None)}
    for k in names:
        gp = tape.grads.get(params[k])
        assert gp is not None, f"{tag}: no gradient for {k}"
        e, c = rell2(gp, osd[k].grad), rell2(csd[k].grad, osd[k].grad)
        key = "wgrad(l2)" if osd[k].dim() == 4 else "bn/bias grad(l2)"
        # rank by how far the engine is above the control
        if e - 1.5 * c > worst[key][0] - 1.5 * worst[key][1] or worst[key][2] is None:
            worst[key] = (e, c, k)
    for key, (e, c, k) in worst.items():
        if k is not None:
            res[f"{key} @{k.replace(prefixes[0], '')}"] = (e, c)
    log(gpu_out_dir, f"{tag} engine|control: " + "  ".join(f"{k} {e:.2e}|{c:.2e}" for k, (e, c) in res.items()))
    bad = []
    for k, (e, c) in res.items():
        tol = FWD_TOL if k.startswith("fwd") else DGRAD_TOL
        if e > max(tol, 1.5 * c):
            bad.append(f"{k} {e:.2e} > max({tol:.0e}, 1.5 x control {c:.2e})")
    return [f"{tag}: {b}" for b in bad]


def test_blocks_c3_deeplab_r101_513(gpu_out_dir):
    nc, backbone, B, S = 19, "resnet101", 4, 513
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    sd = weights.deeplab_resnet_state_dict(nc, backbone, seed=0, randomize_bn=False)
    m = seg_b200.DeepLab(nc, backbone=backbone, pretrained=False, output_stride=16)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m = m.cuda().train()
    x, y = synth.make_batch(B, S, S, nc, 255, seed=9001)
    # ---- oracle full pass, recording block boundaries ----
    osd = om.clone_sd(sd, requires_grad=True)
    rec = Recorder()
    h = om._conv(osd, "backbone.layer0.0", x, 2, 3)
    h = F.relu(om._bn(osd, "backbone.layer0.1", h, True))
    h = F.max_pool2d(h, 3, 2, 1)
    cfg = {1: (1, 1), 2: (2, 1), 3: (2, 1), 4: (1, 2)}
    layers = weights.RESNET_LAYERS[backbone]
    low = None
    for li in (1, 2, 3, 4):
        stride, dil = cfg[li]
        for b in range(layers[li - 1]):
            p = f"backbone.layer{li}.{b}."
            s = stride if b == 0 else 1
            h = _run_block(rec, osd, p, s, dil, h)
        if li == 1:
            low = h
    f = _run(rec, osd, "ASSP.", lambda o, t: om.aspp(o, t, 16, True), h)
    lo = _run(rec, osd, "decoder.", lambda o, a, b_: om.decoder(o, a, b_, True), f, low)
    out = F.interpolate(lo, size=(S, S), mode="bilinear", align_corners=True)
    ol.cross_entropy2d(out, y, 255).backward()
    chosen = {"backbone.layer1.0.", "backbone.layer1.1.", "backbone.layer2.0.", "backbone.layer2.1.", "backbone.layer3.0.",
              "backbone.layer3.1.", "backbone.layer3.22.", "backbone.layer4.0.", "backbone.layer4.1.", "ASSP.", "decoder."}
    failures = []
    for name, fn, inputs, o in rec.steps:
        if name not in chosen:
            continue
        if name.startswith("backbone."):
            li, bi = int(name.split(".")[1][5:]), int(name.split(".")[2])
            blk = getattr(m.backbone, f"layer{li}")[bi]
            eng = (lambda n_, b_: lambda tape, a: m._block(tape, a, n_, b_))(name, blk)
        elif name == "ASSP.":
            eng = lambda tape, a: m._aspp(tape, a)
        else:
            eng = lambda tape, a, b_: m._decoder(tape, a, b_)
        shapes = " ".join("x".join(map(str, t.shape)) for t in inputs)
        failures += check_block(gpu_out_dir, f"[C3 {name} in {shapes}]", fn, [t.detach() for t in inputs], o.grad, eng, m, [name], sd)
    assert not failures, "\n".join(failures)


def _run(rec, osd, name, fn, *inputs):
    out = fn(osd, *inputs)
    out.retain_grad()
    rec.steps.append((name, fn, inputs, out))
    return out


def _run_block(rec, osd, p, s, dil, h, d0=None):
    """One Bottleneck; d0: PSPNet's first-block dilation differs from the rest (models/resnet.py:190-210)."""
    d = dil if d0 is None else d0
    return _run(rec, osd, p, lambda o, t: om._bottleneck(o, p, t, s, d, True), h)


def test_blocks_c2_pspnet_r50_473(gpu_out_dir):
    nc, backbone, B, S = 21, "resnet50", 4, 473
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    sd = weights.pspnet_state_dict(nc, backbone, seed=1, randomize_bn=False)
    m = seg_b200.PSPNet(nc, backbone=backbone, pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    m = m.cuda().train()
    x, y = synth.make_batch(B, S, S, nc, 255, seed=9002)
    osd = om.clone_sd(sd, requires_grad=True)
    rec = Recorder()
    h = F.relu(om._bn(osd, "initial.0.1", om._conv(osd, "initial.0.0", x, 2, 1), True))
    h = F.relu(om._bn(osd, "initial.0.4", om._conv(osd, "initial.0.3", h, 1, 1), True))
    h = F.relu(om._bn(osd, "initial.1", om._conv(osd, "initial.0.6", h, 1, 1), True))
    h = F.max_pool2d(h, 3, 2, 1)
    cfg = {1: (1, 1, 1), 2: (2, 1, 1), 3: (1, 1, 2), 4: (1, 2, 4)}
    layers = weights.RESNET_LAYERS[backbone]
    for li in (1, 2, 3, 4):
        stride, d0, d = cfg[li]
        for b in range(layers[li - 1]):
            h = _run_block(rec, osd, f"layer{li}.{b}.", stride if b == 0 else 1, d, h, d0=d0 if b == 0 else d)

    def head(o, t):
        hh, ww = t.shape[2:]
        pyr = [t]
        for i, bins in enumerate((1, 2, 3, 6)):
            p = F.adaptive_avg_pool2d(t, bins)
            p = F.relu(om._bn(o, f"master_branch.0.stages.{i}.2", om._conv(o, f"master_branch.0.stages.{i}.1", p), True))
            pyr.append(F.interpolate(p, size=(hh, ww), mode="bilinear", align_corners=True))
        yy = om._conv(o, "master_branch.0.bottleneck.0", torch.cat(pyr, 1), 1, 1)
        yy = F.relu(om._bn(o, "master_branch.0.bottleneck.1", yy, True))
        return om._conv(o, "master_branch.1", yy)

    lo = _run(rec, osd, "master_branch.", head, h)
    out = F.interpolate(lo, size=(S, S), mode="bilinear", align_corners=False)
    ol.cross_entropy2d(out, y, 255).backward()
    chosen = {"layer2.0.", "layer3.0.", "layer3.1.", "layer4.0.", "layer4.1.", "master_branch."}
    failures = []
    for name, fn, inputs, o in rec.steps:
        if name not in chosen:
            continue
        if name.startswith("layer"):
            li, bi = int(name.split(".")[0][5:]), int(name.split(".")[1])
            blk = getattr(m, f"layer{li}")[bi]
            eng = (lambda n_, b_: lambda tape, a: m._block(tape, a, n_, b_))(name, blk)
        else:
            eng = lambda tape, a: m._psp_head(tape, a)
        shapes = " ".join("x".join(map(str, t.shape)) for t in inputs)
        failures += check_block(gpu_out_dir, f"[C2 {name} in {shapes}]", fn, [t.detach() for t in inputs], o.grad, eng, m, [name], sd)
    assert not failures, "\n".join(failures)
