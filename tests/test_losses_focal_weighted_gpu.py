"""Cross-entropy, class-weighted cross-entropy and focal loss on the H100 (seg_loss_nchw_*, seg_upsample_loss_*, seg_b200.FocalLoss,
CrossEntropyLoss2d(weight, reduction), FusedTrainStep(loss=...)) against the float64 oracle on the same inputs
(oracle/losses_weighted.py: weighted_loss_and_grad, which tests/test_losses_focal_weighted_cpu.py checks against the reference)."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import losses as ol
from oracle import losses_weighted as olw
from oracle import synth, weights

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import lib, losses, ops
    from seg_b200.train import FusedTrainStep

DEV = "cuda"
GAMMAS = (None, 0.0, 0.5, 1.0, 2.0, 2.5)  # None: class-weighted cross-entropy
CLASSES = ((19, 255), (21, 255), (150, -1))


def log(gpu_out_dir, msg):
    print(msg)
    with open(os.path.join(gpu_out_dir, "losses_focal_weighted.txt"), "a") as f:
        f.write(msg + "\n")


def rel(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def class_weights(C, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(C, generator=g) * 2 + 0.1
    w[torch.randperm(C, generator=g)[: max(2, C // 6)]] = 0.0
    return w


def nchw_inputs(C, ign, special, seed=5):
    g = torch.Generator().manual_seed(seed)
    N, H, W = 2, 33, 37
    z = torch.randn(N, C, H, W, generator=g) * 3
    t = torch.randint(0, C, (N, H, W), generator=g)
    t[:, :3, :] = ign
    t[:, :, -2:] = ign
    w = class_weights(C, seed)
    if special == "img_ignored":
        t[1] = ign
    elif special == "all_ignored":
        t[:] = ign
    elif special == "zero_weight":
        t[t != ign] = int(torch.nonzero(w == 0)[0])
    elif special == "saturated":
        z[:, :, 5:9, :] = 0.0
        z[:, 0, 5:9, :] = 100.0
        t[:, 5:9, :] = 0
    return z, t, w


def engine_nchw(z, t, ign, w, gamma, mean):
    zd, td = z.contiguous().to(DEV), t.to(DEV)
    wd = None if w is None else w.float().to(DEV)
    loss, accum = ops.loss_nchw_fwd(zd, td, ign, wd, gamma, mean)
    dl = ops.loss_nchw_bwd(zd, td, ign, accum, wd, gamma, mean)
    return loss, dl


def raw_wce_nchw(z, t, ign):
    """SEG_LOSS_WCE without class weights, as a mean, through the C ABI: ops runs SEG_LOSS_CE for that combination, so
    this keeps the unit-weight path of the weighted kernels compared with the oracle."""
    zd, td = z.contiguous().to(DEV), t.to(DEV)
    N, C, H, W = zd.shape
    accum = torch.zeros(2, dtype=torch.float64, device=DEV)
    loss = torch.empty((), dtype=torch.float32, device=DEV)
    dl = torch.empty_like(zd)
    lib.call("seg_loss_nchw_fwd", zd.data_ptr(), td.data_ptr(), N, C, H, W, ign, None, lib.LOSS_WCE, 0.0, accum.data_ptr())
    lib.call("seg_loss_finalize", accum.data_ptr(), 1, loss.data_ptr())
    lib.call("seg_loss_nchw_bwd", zd.data_ptr(), td.data_ptr(), N, C, H, W, ign, None, lib.LOSS_WCE, 0.0, 1, accum.data_ptr(),
             None, dl.data_ptr())
    return loss, dl


NCHW_CASES = [(C, ign, gm, use_w, mean, "none") for C, ign in CLASSES for gm in GAMMAS for use_w in (False, True)
              for mean in (True, False)]
NCHW_CASES += [(19, 255, gm, use_w, mean, sp) for sp in ("img_ignored", "all_ignored", "zero_weight", "saturated")
               for gm in (None, 0.0, 0.5, 2.0) for use_w in (False, True) for mean in (True, False)]


@pytest.mark.parametrize("C,ign,gamma,use_w,mean,special", NCHW_CASES)
def test_nchw_matches_oracle(C, ign, gamma, use_w, mean, special, gpu_out_dir):
    z, t, w = nchw_inputs(C, ign, special)
    w = w if use_w else None
    ref_l, ref_g = olw.weighted_loss_and_grad(z, t, ign, None if w is None else w.double(), gamma, mean)
    runs = [("", engine_nchw(z, t, ign, w, gamma, mean))]
    if w is None and gamma is None and mean:
        runs.append((" SEG_LOSS_WCE", raw_wce_nchw(z, t, ign)))
    for suffix, (loss, dl) in runs:
        tag = f"nchw C={C} gamma={gamma} w={use_w} mean={mean} {special}{suffix}"
        assert torch.isfinite(dl).all(), tag
        if float(ref_l) == 0.0 and float(ref_g.abs().max()) == 0.0:  # nothing valid / only zero-weight classes
            assert float(loss) == 0.0 and float(dl.abs().max()) == 0.0, tag
            log(gpu_out_dir, f"{tag}: loss 0, gradient 0")
            continue
        el, eg = abs(float(loss) - float(ref_l)) / abs(float(ref_l)), rel(dl, ref_g)
        log(gpu_out_dir, f"{tag}: loss rel {el:.2e}, grad {eg:.2e}")
        assert el <= 1e-5 and eg <= 1e-4, tag
        if special == "saturated" and gamma is not None and gamma > 0:  # the finite limit, where the reference gives NaN
            assert float(dl.cpu()[:, :, 5:9, :].abs().max()) == 0.0, tag


@pytest.mark.parametrize("C,ign", CLASSES)
def test_focal_gamma0_is_ce_sum_over_all_pixels(C, ign):
    z, t, _ = nchw_inputs(C, ign, "none")
    zd, td = z.to(DEV), t.to(DEV)
    focal = losses.FocalLoss(gamma=0, ignore_index=ign)(zd, td)
    ce_sum = losses.CrossEntropyLoss2d(ignore_index=ign, reduction="sum")(zd, td)
    assert abs(float(focal) - float(ce_sum) / t.numel()) <= 1e-6 * abs(float(focal))


@pytest.mark.parametrize("C,ign", CLASSES)
def test_modules_match_oracle(C, ign, gpu_out_dir):
    """The plugin surface: CrossEntropyLoss2d(weight, reduction), FocalLoss(gamma, alpha, size_average) and
    CE_DiceLoss(weight) through autograd, with an upstream gradient."""
    z, t, w = nchw_inputs(C, ign, "none", seed=9)
    t_nd = t.clone()
    t_nd[t_nd == ign] = 1  # CE_DiceLoss on a target without ignored pixels (the reference's Dice rewrites ignored labels)
    mods = [("ce_w_mean", losses.CrossEntropyLoss2d(weight=w.tolist(), ignore_index=ign), (w, None, True), t),
            ("ce_sum", losses.CrossEntropyLoss2d(ignore_index=ign, reduction="sum"), (None, None, False), t),
            ("focal", losses.FocalLoss(ignore_index=ign), (None, 2.0, True), t),
            ("focal_alpha_sum", losses.FocalLoss(gamma=1.5, alpha=w, ignore_index=ign, size_average=False), (w, 1.5, False), t),
            ("ce_dice_w", losses.CE_DiceLoss(weight=w, ignore_index=ign), (w, None, True), t_nd)]
    for name, mod, (ww, gm, mean), tt in mods:
        x = z.clone().to(DEV).requires_grad_(True)
        loss = mod(x, tt.clone().to(DEV))
        (0.7 * loss).backward()
        ref_l, ref_g = olw.weighted_loss_and_grad(z, tt, ign, None if ww is None else ww.double(), gm, mean)
        if name == "ce_dice_w":
            xr = z.double().clone().requires_grad_(True)
            d = ol.dice_loss(xr, tt.clone())
            d.backward()
            ref_l, ref_g = ref_l + d.detach(), ref_g + xr.grad
        el, eg = abs(float(loss.detach()) - float(ref_l)) / abs(float(ref_l)), rel(x.grad, 0.7 * ref_g)
        log(gpu_out_dir, f"module {name} C={C}: loss rel {el:.2e}, grad {eg:.2e}")
        assert el <= 1e-5 and eg <= 1e-4, name
    with pytest.raises(ValueError):
        losses.CrossEntropyLoss2d(weight=[1.0] * (C + 1), ignore_index=ign)(z.to(DEV), t.to(DEV))


def fused_inputs(N, C, ign, Hi, Wi, Ho, Wo, special, seed=11):
    g = torch.Generator().manual_seed(seed)
    lo = torch.randn(N, C, Hi, Wi, generator=g) * 3
    t = torch.randint(0, C, (N, Ho, Wo), generator=g)
    t[:, :4, :] = ign
    w = class_weights(C, seed)
    if special == "all_ignored":
        t[:] = ign
    elif special == "zero_weight":
        t[t != ign] = int(torch.nonzero(w == 0)[0])
    return lo, t, w


def fused_oracle(lo, t, ign, w, gamma, mean, ac):
    """float64 on the device: upsample, the engine's loss definition, and the gradient back through the upsample."""
    x = lo.to(DEV).double().requires_grad_(True)
    full = F.interpolate(x, size=t.shape[1:], mode="bilinear", align_corners=ac)
    l, g = olw.weighted_loss_and_grad(full.detach(), t.to(DEV), ign, None if w is None else w.double(), gamma, mean)
    full.backward(g)
    return l, x.grad


FUSED_SHAPES = {"small": (2, 17, 19, 65, 73), "c3": (16, 129, 129, 513, 513), "c5": (8, 128, 128, 512, 512)}
FUSED_CASES = [("small", C, ign, gm, use_w, mean, ac, "none") for C, ign in ((19, 255), (150, -1)) for gm in (None, 0.5, 2.0)
               for use_w in (False, True) for mean in (True, False) for ac in (True, False)]
FUSED_CASES += [("small", 19, 255, gm, True, True, ac, sp) for sp in ("all_ignored", "zero_weight") for gm in (None, 2.0)
                for ac in (True, False)]
FUSED_CASES += [("c3", 19, 255, 2.0, True, True, True, "none"), ("c3", 19, 255, None, True, True, False, "none"),
                ("c5", 150, -1, 2.0, False, True, False, "none"), ("c5", 150, -1, None, True, False, True, "none")]


@pytest.mark.parametrize("shape,C,ign,gamma,use_w,mean,ac,special", FUSED_CASES)
def test_fused_upsample_loss(shape, C, ign, gamma, use_w, mean, ac, special, gpu_out_dir):
    N, Hi, Wi, Ho, Wo = FUSED_SHAPES[shape]
    lo, t, w = fused_inputs(N, C, ign, Hi, Wi, Ho, Wo, special)
    w = w if use_w else None
    lod = lo.permute(0, 2, 3, 1).contiguous().to(DEV)
    td = t.to(DEV)
    wd = None if w is None else w.float().to(DEV)
    ldx = (C + 7) // 8 * 8
    runs = []
    for _ in range(2):
        loss, accum, _ = ops.upsample_loss_fwd(lod, td, ac, ign, wd, gamma, mean)
        dx, dlo = ops.upsample_loss_bwd(lod, td, ac, ign, accum, ldx, wd, gamma, mean)
        runs.append((loss.clone(), dlo.clone(), dx.clone()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1])), "two runs differ"
    loss, dlo, dx = runs[0]
    tag = f"fused {shape} C={C} gamma={gamma} w={use_w} mean={mean} ac={ac} {special}"
    if special != "none":  # nothing valid, or only zero-weight classes present
        assert float(loss) == 0.0 and float(dlo.abs().max()) == 0.0 and float(dx.float().abs().max()) == 0.0, tag
        log(gpu_out_dir, f"{tag}: loss 0, gradient 0")
        return
    ref_l, ref_g = fused_oracle(lo, t, ign, w, gamma, mean, ac)
    ref_g = ref_g.permute(0, 2, 3, 1)
    el = abs(float(loss) - float(ref_l)) / abs(float(ref_l))
    e32, e16 = rel(dlo, ref_g), rel(dx[..., :C].float(), ref_g)
    log(gpu_out_dir, f"{tag}: loss rel {el:.2e}, dlo {e32:.2e}, dx(bf16) {e16:.2e}")
    assert el <= 1e-5 and e32 <= 1e-4 and e16 <= 1e-2, tag
    assert float(dx[..., C:].float().abs().max() if ldx > C else 0.0) == 0.0


def _model(kind, seed):
    if kind == "deeplab":
        sd = weights.deeplab_resnet_state_dict(7, "resnet14", seed=seed, randomize_bn=True)
        m = seg_b200.DeepLab(7, backbone="resnet14", pretrained=False, output_stride=16)
    else:
        sd = weights.pspnet_state_dict(7, "resnet14", seed=seed, randomize_bn=True)
        m = seg_b200.PSPNet(7, backbone="resnet14", pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    return m.cuda().train()


def _heads(out):
    return out if isinstance(out, tuple) else (out, None)


@pytest.mark.parametrize("kind", ["deeplab", "pspnet"])
def test_plugin_focal_backward_matches_torch_formula(kind, gpu_out_dir):
    """FocalLoss()(model(x), y).backward() (PSPNet: + 0.4 x the aux head, trainer.py:57-61) gives the parameter gradients
    that the reference formula, applied with torch autograd to the same logits, gives through the same engine backward."""
    m = _model(kind, 21)
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9021)
    xd, yd = x.cuda(), y.cuda()
    grads = []
    for use_engine in (True, False):
        for p in m.parameters():
            p.grad = None
        out, aux = _heads(m(xd))
        if use_engine:
            crit = seg_b200.FocalLoss(ignore_index=255)
        else:
            crit = lambda o, t: olw.focal_loss(o, t, gamma=2, ignore_index=255)  # noqa: E731
        loss = crit(out, yd) + (0.4 * crit(aux, yd) if aux is not None else 0.0)
        loss.backward()
        grads.append(torch.cat([p.grad.detach().reshape(-1).double() for p in m.parameters()]))
    e = rel(grads[0], grads[1])
    cos = float(F.cosine_similarity(grads[0], grads[1], dim=0))
    log(gpu_out_dir, f"plugin focal {kind}: parameter-gradient rel {e:.2e}, cosine {cos:.7f}")
    assert e <= 1e-2 and cos > 0.99999


def _spec_losses():
    w = class_weights(7, 3).tolist()
    return {"ce_w": lambda: losses.CrossEntropyLoss2d(weight=w, ignore_index=255),
            "ce_sum": lambda: losses.CrossEntropyLoss2d(ignore_index=255, reduction="sum"),
            "focal": lambda: losses.FocalLoss(ignore_index=255),
            "focal_alpha_sum": lambda: losses.FocalLoss(gamma=0.5, alpha=w, ignore_index=255, size_average=False)}


@pytest.mark.parametrize("kind", ["deeplab", "pspnet"])
@pytest.mark.parametrize("name", ["ce_w", "ce_sum", "focal", "focal_alpha_sum"])
def test_fused_step_first_loss_equals_plugin(kind, name, gpu_out_dir):
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9022)
    xd, yd = x.cuda(), y.cuda()
    crit = _spec_losses()[name]()
    m = _model(kind, 22)
    with torch.no_grad():
        out, aux = _heads(m(xd))
        ref = float(crit(out, yd) + (0.4 * crit(aux, yd) if aux is not None else 0.0))
    m = _model(kind, 22)
    got = float(FusedTrainStep(m, lr=0.005, loss=crit).step(xd, yd))
    log(gpu_out_dir, f"fused step [{kind} {name}] first loss {got:.7f}, plugin {ref:.7f}")
    assert abs(got - ref) <= 1e-4 * abs(ref)


@pytest.mark.parametrize("name", ["ce_w", "focal", "focal_alpha_sum"])
def test_fused_step_graph_replay_equals_eager(name, gpu_out_dir):
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9023)
    xd, yd = x.cuda(), y.cuda()
    crit = _spec_losses()[name]()
    m_e, m_g = _model("pspnet", 23), _model("pspnet", 23)
    se, sg = FusedTrainStep(m_e, lr=0.005, loss=crit), FusedTrainStep(m_g, lr=0.005, loss=crit, cuda_graph=True)
    for i in range(3):
        le, lg = float(se.step(xd, yd)), float(sg.step(xd, yd))
        log(gpu_out_dir, f"graph-vs-eager [{name}] step {i}: eager {le:.7f} graph {lg:.7f}")
        assert le == le and abs(le - lg) <= 1e-5 * abs(le), (i, le, lg)
    assert sg.steps == 3
    sg.release_graph()


def test_fused_step_with_plain_ce_is_bit_identical_to_default():
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9024)
    xd, yd = x.cuda(), y.cuda()
    ms = [_model("pspnet", 24) for _ in range(2)]
    steppers = [FusedTrainStep(ms[0], lr=0.005), FusedTrainStep(ms[1], lr=0.005, loss=losses.CrossEntropyLoss2d())]
    ls = [[float(s.step(xd, yd)) for _ in range(2)] for s in steppers]
    assert ls[0] == ls[1]
    assert torch.equal(steppers[0].flat_grad, steppers[1].flat_grad)
    for a, b in zip(ms[0].parameters(), ms[1].parameters()):
        assert torch.equal(a, b)


def test_fused_step_rejects_unsupported_losses():
    m = _model("deeplab", 25)
    for crit in (losses.DiceLoss(), losses.CE_DiceLoss(), losses.LovaszSoftmax()):
        with pytest.raises(NotImplementedError, match="plugin surface"):
            FusedTrainStep(m, loss=crit)
    with pytest.raises(ValueError):
        FusedTrainStep(m, ignore_index=255, loss=losses.FocalLoss(ignore_index=-1))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_global_batch_losses(tmp_path):
    """Weighted and focal losses under torchrun with unequal valid-pixel counts per rank equal one GPU on the whole batch."""
    out = tmp_path / "dp_losses.txt"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", "29613", os.path.join(root, "tests", "losses_dp_worker.py"), str(out)],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert out.read_text().strip().endswith("ok")
