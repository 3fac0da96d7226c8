"""DeepLab_DUC_HDC on the H100: the pixel-shuffle kernels (seg_pixel_shuffle_*, seg_pixel_shuffle_logits_*) against
F.pixel_shuffle bit for bit, the fused shuffle + loss kernels (seg_shuffle_loss_*) against the float64 oracle of
oracle/losses_weighted.py and against seg_eval_metrics_nchw, the model against the fp32 oracle of oracle/duc_hdc.py (pinned to
the reference by tests/golden/duc_hdc.npz), and FusedTrainStep through the shuffle head."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import duc_hdc as od
from oracle import losses as ol
from oracle import losses_weighted as olw
from oracle import models as om
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import losses, ops
    from seg_b200.train import FusedTrainStep

DEV = "cuda"


def log(gpu_out_dir, msg):
    print(msg)
    with open(os.path.join(gpu_out_dir, "duc_hdc.txt"), "a") as f:
        f.write(msg + "\n")


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def cosine(a, b):
    return F.cosine_similarity(a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten(), dim=0).item()


def pitched(t, lead, trail, fill=7.0):
    """t [..., C] copied into the middle of a wider guard-filled device buffer: (channel slice with its own pitch, buffer)."""
    C = t.shape[-1]
    buf = torch.full(t.shape[:-1] + (lead + C + trail,), fill, dtype=t.dtype, device=DEV)
    buf[..., lead:lead + C] = t.to(DEV)
    return buf[..., lead:lead + C], buf


def guards_intact(buf, lead, C, fill=7.0):
    return bool((buf[..., :lead] == fill).all() and (buf[..., lead + C:] == fill).all())


# ------------------------------------------------------------------------------------------------ pixel shuffle
@pytest.mark.parametrize("r", [2, 4])
@pytest.mark.parametrize("crop", [False, True], ids=["full", "cropped"])
def test_pixel_shuffle_exact(r, crop):
    g = torch.Generator().manual_seed(10 * r + crop)
    N, H, W, C = 2, 5, 7, 6
    Ho, Wo = (r * H - 1, r * W - r - 1) if crop else (r * H, r * W)
    x, _ = pitched(torch.randn(N, H, W, C * r * r, generator=g).bfloat16(), 8, 16)
    y, ybuf = pitched(torch.zeros(N, Ho, Wo, C, dtype=torch.bfloat16), 3, 5)
    ops.pixel_shuffle_fwd(x, r, Ho, Wo, out=y)
    ref = F.pixel_shuffle(x.float().permute(0, 3, 1, 2).cpu(), r)[:, :, :Ho, :Wo].permute(0, 2, 3, 1)
    assert torch.equal(y.float().cpu(), ref) and guards_intact(ybuf, 3, C)
    # backward: the inverse permutation; positions the crop dropped get zero; beta = 1 accumulates
    dy, _ = pitched(torch.randn(N, Ho, Wo, C, generator=g).bfloat16(), 8, 8)
    xin = torch.zeros(N, C * r * r, H, W, requires_grad=True)
    F.pixel_shuffle(xin, r)[:, :, :Ho, :Wo].backward(dy.float().permute(0, 3, 1, 2).cpu())
    want = xin.grad.permute(0, 2, 3, 1)
    dx, dxbuf = pitched(torch.zeros(N, H, W, C * r * r, dtype=torch.bfloat16), 8, 8)
    ops.pixel_shuffle_bwd(dy, r, H, W, dx=dx, beta=0.0)
    assert torch.equal(dx.float().cpu(), want) and guards_intact(dxbuf, 8, C * r * r)
    prev = torch.randn(N, H, W, C * r * r, generator=g).bfloat16()
    dx.copy_(prev.to(DEV))
    ops.pixel_shuffle_bwd(dy, r, H, W, dx=dx, beta=1.0)
    assert torch.equal(dx.cpu(), (prev.float() + want).bfloat16()) and guards_intact(dxbuf, 8, C * r * r)


@pytest.mark.parametrize("r", [2, 4])
def test_pixel_shuffle_logits_exact(r):
    g = torch.Generator().manual_seed(r)
    N, h, w, C = 2, 6, 5, 19
    x, _ = pitched(torch.randn(N, h, w, C * r * r, generator=g).bfloat16(), 0, 8)
    y = ops.pixel_shuffle_logits_fwd(x, r)
    assert torch.equal(y.cpu(), F.pixel_shuffle(x.float().permute(0, 3, 1, 2).cpu(), r))
    dy = torch.randn(N, C, h * r, w * r, generator=g)
    ldx = (C * r * r + 7) // 8 * 8 + 8
    dx = ops.pixel_shuffle_logits_bwd(dy.to(DEV), r, ldx)
    assert torch.equal(dx[..., : C * r * r].cpu(), F.pixel_unshuffle(dy, r).permute(0, 2, 3, 1).bfloat16())
    assert (dx[..., C * r * r:] == 0).all()


# ------------------------------------------------------------------------------------------------ shuffle + loss
def class_weights(C, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(C, generator=g) * 2 + 0.1
    w[torch.randperm(C, generator=g)[: max(2, C // 6)]] = 0.0
    return w


def shuffle_inputs(C, r, ign, special, seed):
    g = torch.Generator().manual_seed(seed)
    N, h, w = 2, 5, 6
    lo = (torch.randn(N, h, w, C * r * r, generator=g) * 3).bfloat16()
    t = torch.randint(0, C, (N, h * r, w * r), generator=g)
    t[:, :3, :] = ign
    t[:, :, -2:] = ign
    wts = class_weights(C, seed)
    if special == "all_ignored":
        t[:] = ign
    elif special == "zero_weight":
        t[t != ign] = int(torch.nonzero(wts == 0)[0])
    return lo, t, wts


# (name, weighted, gamma, mean)
LOSSES = [("ce", False, None, True), ("wce", True, None, True), ("wce_sum", True, None, False), ("focal0", False, 0.0, True),
          ("focal0.5_w", True, 0.5, True), ("focal2", False, 2.0, True), ("focal2_w_sum", True, 2.0, False)]


@pytest.mark.parametrize("C,ign", [(7, 255), (19, 255), (150, -1)])
@pytest.mark.parametrize("special", ["plain", "zero_weight", "all_ignored"])
def test_shuffle_loss_matches_oracle(C, ign, special, gpu_out_dir):
    worst = (0.0, 0.0)
    for r in (2, 4):
        lo, t, wts = shuffle_inputs(C, r, ign, special, seed=C + r)
        lod, td = pitched(lo, 0, 8)[0], t.to(DEV)
        z = F.pixel_shuffle(lo.float().permute(0, 3, 1, 2), r)
        ldx = (C * r * r + 7) // 8 * 8
        for name, weighted, gamma, mean in LOSSES:
            w = wts if weighted else None
            wd = None if w is None else w.to(DEV)
            loss, accum = ops.shuffle_loss_fwd(lod, r, td, ign, wd, gamma, mean)
            dx = ops.shuffle_loss_bwd(lod, r, td, ign, accum, ldx, wd, gamma, mean)
            ref_loss, ref_grad = olw.weighted_loss_and_grad(z, t, ign, w, gamma, mean)
            got = F.pixel_shuffle(dx[..., : C * r * r].float().permute(0, 3, 1, 2).cpu(), r).double()
            assert (dx[..., C * r * r:] == 0).all()
            le = abs(loss.item() - ref_loss.item()) / max(abs(ref_loss.item()), 1e-30)
            scale = ref_grad.abs().max().item()
            # the gradient is formed in fp32 and stored in bf16: one bf16 rounding on top of the fp32 bound
            excess = ((got - ref_grad).abs() - 2.0 ** -8 * ref_grad.abs()).max().item() / max(scale, 1e-30)
            assert le <= 1e-6 or abs(ref_loss.item()) < 1e-30 and loss.item() == 0.0, (r, name, le)
            assert excess <= 1e-5, (r, name, excess)
            if special == "all_ignored" and mean and gamma is None:
                assert loss.item() == 0.0 and (dx == 0).all()
            worst = max(worst, (le, excess))
    log(gpu_out_dir, f"shuffle loss C={C} ignore={ign} {special}: worst loss rel {worst[0]:.2e}, grad excess {worst[1]:.2e}")


@pytest.mark.parametrize("C", [7, 19, 150])
def test_shuffle_loss_counters_equal_eval_metrics(C):
    """The counters of the fused forward equal seg_eval_metrics_nchw on the shuffled logits exactly, including planted ties
    (lowest index wins) and pixels whose scores are all zero (as ReLU'd DUC_out scores often are); two runs are bit-identical."""
    r = 4
    lo, t, _ = shuffle_inputs(C, r, 255, "plain", seed=40 + C)
    t[0, 5:9, 5:9] = 3 % C
    lo[0, 1, 1, :] = 0.0                                     # all-zero low-res pixel: 16 full-res pixels, every class 0
    lo[1, 2, 3, 5 * 16:6 * 16] = lo[1, 2, 3].reshape(C, 16).max(0).values  # classes 2 and 5 tie at the top at 16 pixels
    lo[1, 2, 3, 2 * 16:3 * 16] = lo[1, 2, 3, 5 * 16:6 * 16]
    t[1, 8:12, 12:16] = 5
    lod, td = lo.to(DEV), t.to(DEV)
    want = ops.eval_metrics_nchw(ops.pixel_shuffle_logits_fwd(lod, r), td, C)
    runs = []
    for _ in range(2):
        cnt = torch.zeros(2 + 3 * C, dtype=torch.int64, device=DEV)
        loss, accum = ops.shuffle_loss_fwd(lod, r, td, 255, counters=cnt)
        dx = ops.shuffle_loss_bwd(lod, r, td, 255, accum, (C * r * r + 7) // 8 * 8)
        runs.append((loss.clone(), accum.clone(), dx.clone(), cnt))
    assert torch.equal(runs[0][3], want), (runs[0][3].tolist(), want.tolist())
    assert int(want[1]) > 0 and int(want[0]) > 0
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)


def test_shuffle_loss_rejects_a_target_of_another_size():
    lo = torch.zeros(1, 4, 4, 16 * 7, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(ValueError, match=r"\(15, 16\).*\(16, 16\)"):
        ops.shuffle_loss_fwd(lo, 4, torch.zeros(1, 15, 16, dtype=torch.int64, device=DEV), 255)


# ------------------------------------------------------------------------------------------------ model vs oracle
def build(nc, seed, **kw):
    sd = od.duc_hdc_state_dict(nc, seed=seed, randomize_bn=True)
    m = seg_b200.DeepLab_DUC_HDC(nc, pretrained=False, **kw)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    return sd, m.cuda()


def argmax_report(gpu_out_dir, tag, out, ref):
    """Argmax agreement; pixels whose top-2 margin is within twice the max error are undecidable (ReLU'd scores tie often)."""
    err = (out.detach().cpu() - ref).abs().max().item()
    top2 = ref.topk(2, dim=1).values
    safe = (top2[:, 0] - top2[:, 1]) > 2 * err
    am_e, am_r = out.detach().argmax(1).cpu(), ref.argmax(1)
    agree_all = (am_e == am_r).float().mean().item()
    agree_safe = (am_e[safe] == am_r[safe]).float().mean().item() if safe.any() else 1.0
    log(gpu_out_dir, f"{tag} argmax vs oracle: all pixels {agree_all:.5f}; decidable pixels ({safe.float().mean().item():.3f} of map) {agree_safe:.5f}")
    return agree_all, agree_safe


@pytest.mark.parametrize("os_,size", [(8, 64), (4, 32)])
def test_frozen_bn_train_step_parity(os_, size, gpu_out_dir):
    """Frozen BatchNorm: every forward and backward kernel in context (the shuffle head, the DUC shuffle into the concat
    buffer, the data gradient of DUC_out's im2col conv) against the fp32 oracle at the bf16 noise floor."""
    sd, m = build(19, 11, output_stride=os_)
    x, y = synth.make_batch(2, size, size, 19, 255, seed=9031)
    y = F.interpolate(y[:, None].float(), size=(size * 8 // os_, size * 8 // os_), mode="nearest")[:, 0].long()
    osd = om.clone_sd(sd, requires_grad=True)
    ref = od.duc_hdc_forward(osd, x, output_stride=os_, train=False)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    m.train()
    m.freeze_bn()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[frozen-BN duc_hdc os{os_}]"
    e = relerr(out, ref)
    log(gpu_out_dir, f"{tag} logits rel_err vs fp32 oracle {e:.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert out.shape == ref.shape and e < 5e-2
    assert abs(loss.item() - ref_loss.item()) < 1e-2 * abs(ref_loss.item())
    _, agree_safe = argmax_report(gpu_out_dir, tag, out, ref.detach())
    assert agree_safe == 1.0
    cos_min, cos_name = 1.0, None
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        if osd[name].grad.abs().max() == 0:
            continue
        c = cosine(p.grad, osd[name].grad)
        if c < cos_min:
            cos_min, cos_name = c, name
    log(gpu_out_dir, f"{tag} grads vs fp32 oracle: min cosine {cos_min:.5f} at {cos_name}")
    assert cos_min > 0.9, (cos_min, cos_name)
    esd = m.state_dict()
    assert all(torch.equal(esd[k].cpu(), sd[k]) for k in esd if "running_" in k)


def test_eval_forward_and_batchstat_train_step(gpu_out_dir):
    """Eval forward (running statistics) at the bf16 noise floor; then a batch-statistics step, whose 101-layer trunk at
    initialisation amplifies rounding differences (tests/test_model_gpu.py): loss, stem running statistics, finiteness."""
    sd, m = build(19, 12)
    x, y = synth.make_batch(2, 64, 64, 19, 255, seed=9032)
    osd = om.clone_sd(sd, requires_grad=True)
    m.eval()
    with torch.no_grad():
        ev = m(x.cuda())
        ev_ref = od.duc_hdc_forward(osd, x, train=False)
    log(gpu_out_dir, f"[eval duc_hdc] logits rel_err vs fp32 oracle {relerr(ev, ev_ref):.3e}")
    assert ev.shape == ev_ref.shape and relerr(ev, ev_ref) < 5e-2
    ref = od.duc_hdc_forward(osd, x, train=True)
    ref_loss = ol.cross_entropy2d(ref, y, 255)
    ref_loss.backward()
    m.train()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = "[batch-stat duc_hdc os8]"
    log(gpu_out_dir, f"{tag} logits rel_err {relerr(out, ref):.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert abs(loss.item() - ref_loss.item()) < 0.05 * abs(ref_loss.item())
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
    esd = m.state_dict()
    for k in ("backbone.layer0.1.running_mean", "backbone.layer0.1.running_var"):
        assert relerr(esd[k], osd[k]) < 1e-2, k
    assert all(int(esd[k]) == 1 for k in esd if k.endswith("num_batches_tracked"))


# ------------------------------------------------------------------------------------------------ FusedTrainStep
def _model(seed, nc=7):
    m = seg_b200.DeepLab_DUC_HDC(nc, pretrained=False)
    m.load_state_dict(od.duc_hdc_state_dict(nc, seed=seed, randomize_bn=True), strict=True)
    m.engine_dropout = False
    return m.cuda().train()


@pytest.mark.parametrize("name", ["ce", "focal"])
def test_fused_step_first_loss_equals_plugin(name, gpu_out_dir):
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9033)
    xd, yd = x.cuda(), y.cuda()
    crit = losses.CrossEntropyLoss2d(ignore_index=255) if name == "ce" else losses.FocalLoss(ignore_index=255)
    with torch.no_grad():
        ref = float(crit(_model(41)(xd), yd))
    got = float(FusedTrainStep(_model(41), lr=0.005, loss=crit).step(xd, yd))
    log(gpu_out_dir, f"fused step [duc_hdc {name}] first loss {got:.7f}, plugin {ref:.7f}")
    assert abs(got - ref) <= 1e-5 * abs(ref)


def test_fused_step_graph_replay_is_bit_identical_and_counts_like_eval_metrics():
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9034)
    xd, yd = x.cuda(), y.cuda()
    with torch.no_grad():
        want = ops.eval_metrics_nchw(_model(42)(xd), yd, 7)  # the plugin output of the same train-mode forward
    se = FusedTrainStep(_model(42), lr=0.005, metrics=True)
    sg = FusedTrainStep(_model(42), lr=0.005, metrics=True, cuda_graph=True)
    for i in range(3):
        le, lg = float(se.step(xd, yd)), float(sg.step(xd, yd))
        assert le == le and le == lg, (i, le, lg)
        if i == 0:
            assert torch.equal(se.seg_counters, want) and torch.equal(sg.seg_counters, want)
    assert torch.equal(se.flat_grad, sg.flat_grad)
    for (n, a), (_, b) in zip(se.model.state_dict().items(), sg.model.state_dict().items()):
        assert torch.equal(a, b), n
    sg.release_graph()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_evaluate_changes_no_training_state(graph):
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9035)
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
    """A 65x65 input gives a 68x68 output (duc_hdc.py:233); a 65x65 target cannot be scored against it."""
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9036)
    s = FusedTrainStep(_model(44), lr=0.005)
    for call in (s.step, s.evaluate):
        with pytest.raises(ValueError, match=r"\(65, 65\).*\(68, 68\)"):
            call(x.cuda(), y.cuda())


def test_plugin_losses_on_the_output():
    """Dice, CE + Dice and Lovasz (plugin surface) run unchanged on the NCHW output and back-propagate."""
    x, y = synth.make_batch(2, 64, 64, 7, 255, seed=9037)
    y[y == 255] = 0
    m = _model(45)
    for crit in (losses.DiceLoss(), losses.CE_DiceLoss(), losses.LovaszSoftmax()):
        for p in m.parameters():
            p.grad = None
        loss = crit(m(x.cuda()), y.cuda())
        loss.backward()
        assert torch.isfinite(loss) and all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())


def test_full_size_graph_step(gpu_out_dir):
    """One 8 x 3 x 512 x 512 fused graph step (the configs' crop and batch) completes with a finite loss."""
    x, y = synth.make_batch(8, 512, 512, 19, 255, seed=9038)
    s = FusedTrainStep(_model(46, nc=19), lr=0.01, cuda_graph=True)
    loss = float(s.step(x.cuda(), y.cuda()))
    torch.cuda.synchronize()
    log(gpu_out_dir, f"[duc_hdc 8x3x512x512 graph step] loss {loss:.6f}")
    assert loss == loss and abs(loss) < 1e3
    s.release_graph()
