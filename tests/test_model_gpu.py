"""Whole-model GPU parity against the CPU oracle (pinned to the reference by tests/golden).

A random-initialised ~100-layer BatchNorm network in TRAIN mode is chaotic: measured on this engine, two bf16
implementations that differ only in fp32 summation order (wgmma vs CUDA-core kernels) already differ by ~2e-2 in the
logits in eval mode, and batch-statistics BN on small maps amplifies any rounding difference by ~1.3x per residual
block.  So whole-model parity is decomposed into links that can each be checked tightly:

  reference == oracle                       exact   tests/test_oracle_golden.py (golden vectors from the reference itself)
  oracle == engine host logic               ~2e-3   tests/test_engine_cpu_emulated.py (ATen kernel emulation, fp32 storage)
  every kernel == ATen op                   ~1e-6   tests/test_ops_gpu.py (fp32 outputs; bf16 outputs to 1 ulp)
  kernels IN CONTEXT, well-conditioned net  here    frozen-BN train step + eval forward vs the fp32 oracle (bf16 noise floor)
  kernels IN CONTEXT, batch-stat BN         here    loss / running stats / finiteness vs the oracle + the 3-way error log
  optimisation works                        here    over-fitting one batch drives the loss down like the oracle does
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import losses as ol
from oracle import models as om
from oracle import synth, weights

if torch.cuda.is_available():
    import seg_b200
    from seg_b200.lib import IMPL_SIMT
    from seg_b200.train import FusedTrainStep


def log(gpu_out_dir, msg):
    print(msg)
    with open(os.path.join(gpu_out_dir, "model_parity.txt"), "a") as f:
        f.write(msg + "\n")


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def cosine(a, b):
    return torch.nn.functional.cosine_similarity(a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten(), dim=0).item()


def build(kind, nc, backbone, seed, **kw):
    if kind == "deeplab" and backbone == "xception":
        sd = weights.deeplab_xception_state_dict(nc, seed=seed, randomize_bn=True, **kw)
        m = seg_b200.DeepLab(nc, backbone=backbone, pretrained=False, **kw)
    elif kind == "deeplab":
        sd = weights.deeplab_resnet_state_dict(nc, backbone, seed=seed, randomize_bn=True)
        m = seg_b200.DeepLab(nc, backbone=backbone, pretrained=False, **kw)
    elif kind == "upernet":
        sd = weights.upernet_state_dict(nc, backbone, seed=seed, randomize_bn=True)
        m = seg_b200.UperNet(nc, backbone=backbone, pretrained=False, **kw)
    else:
        sd = weights.pspnet_state_dict(nc, backbone, seed=seed, randomize_bn=True)
        m = seg_b200.PSPNet(nc, backbone=backbone, pretrained=False, **kw)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    return sd, m.cuda()


def oracle_forward(kind, osd, x, backbone, kw, train):
    if kind == "deeplab":
        return om.deeplab_forward(osd, x, backbone=backbone, train=train, **kw), None
    if kind == "upernet":
        return om.upernet_forward(osd, x, backbone=backbone, train=train), None
    out = om.pspnet_forward(osd, x, backbone=backbone, train=train)
    return out if isinstance(out, tuple) else (out, None)


CASES = [
    ("deeplab", 19, "resnet101", 0, dict(output_stride=16), 9001),
    ("deeplab", 19, "resnet50", 2, dict(output_stride=8), 9001),
    ("pspnet", 21, "resnet50", 1, dict(), 9002),
    ("upernet", 150, "resnet50", 3, dict(), 9004),
    ("deeplab", 19, "xception", 4, dict(output_stride=16), 9001),
]
IDS = ["deeplab_r101_os16", "deeplab_r50_os8", "pspnet_r50", "upernet_r50", "deeplab_xception_os16"]


def argmax_report(gpu_out_dir, tag, out, ref):
    err = (out.detach().cpu() - ref).abs().max().item()
    top2 = ref.topk(2, dim=1).values
    safe = (top2[:, 0] - top2[:, 1]) > 2 * err
    am_e, am_r = out.detach().argmax(1).cpu(), ref.argmax(1)
    agree_all = (am_e == am_r).float().mean().item()
    agree_safe = (am_e[safe] == am_r[safe]).float().mean().item() if safe.any() else 1.0
    log(gpu_out_dir, f"{tag} argmax vs oracle: all pixels {agree_all:.5f}; pixels with top-2 margin > 2*max_err ({safe.float().mean().item():.3f} of map) {agree_safe:.5f}")
    return agree_all, agree_safe


@pytest.mark.parametrize("kind,nc,backbone,seed,kw,xseed", CASES, ids=IDS)
def test_frozen_bn_train_step_parity(kind, nc, backbone, seed, kw, xseed, gpu_out_dir):
    """BN frozen (BaseModel.freeze_bn, config arch.args.freeze_bn) -> a fixed, well-conditioned function: every forward
    and backward kernel runs in context and can be compared with the fp32 oracle at the bf16 noise floor."""
    sd, m = build(kind, nc, backbone, seed, **kw)
    x, y = synth.make_batch(2, 97, 97, nc, 255, seed=xseed)
    osd = om.clone_sd(sd, requires_grad=True)
    ref_out, _ = oracle_forward(kind, osd, x, backbone, kw, train=False)
    ref_loss = ol.cross_entropy2d(ref_out, y, 255)
    ref_loss.backward()
    m.train()
    m.freeze_bn()
    crit = seg_b200.CrossEntropyLoss2d(ignore_index=255)
    out = m(x.cuda())
    out = out[0] if isinstance(out, tuple) else out
    loss = crit(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[frozen-BN {kind}/{backbone}{kw}]"
    e = relerr(out, ref_out)
    log(gpu_out_dir, f"{tag} logits rel_err vs fp32 oracle {e:.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert e < 5e-2
    assert abs(loss.item() - ref_loss.item()) < 1e-2 * abs(ref_loss.item())
    agree_all, agree_safe = argmax_report(gpu_out_dir, tag, out, ref_out.detach())
    assert agree_safe == 1.0 and agree_all > 0.97
    cos_min, cos_name, n_checked = 1.0, None, 0
    for name, p in m.named_parameters():
        rg = osd[name].grad
        if rg is None:  # aux branch is unused in this mode
            continue
        assert p.grad is not None, f"no grad for {name}"
        assert torch.isfinite(p.grad).all(), name
        if rg.abs().max() == 0:
            continue
        c = cosine(p.grad, rg)
        n_checked += 1
        if c < cos_min:
            cos_min, cos_name = c, name
    log(gpu_out_dir, f"{tag} grads vs fp32 oracle over {n_checked} tensors: min cosine {cos_min:.5f} at {cos_name}")
    assert cos_min > 0.9, f"gradient mismatch (min cosine {cos_min} at {cos_name})"
    # running statistics must be untouched by a frozen-BN step
    esd = m.state_dict()
    assert all(torch.equal(esd[k].cpu(), sd[k]) for k in esd if "running_" in k)


@pytest.mark.parametrize("kind,nc,backbone,seed,kw,xseed", CASES, ids=IDS)
def test_batchstat_train_step(kind, nc, backbone, seed, kw, xseed, gpu_out_dir):
    sd, m = build(kind, nc, backbone, seed, **kw)
    x, y = synth.make_batch(4, 129, 129, nc, 255, seed=xseed)
    osd = om.clone_sd(sd, requires_grad=True)
    ref_out, ref_aux = oracle_forward(kind, osd, x, backbone, kw, train=True)
    ref_loss = ol.cross_entropy2d(ref_out, y, 255)
    if ref_aux is not None:
        ref_loss = ref_loss + 0.4 * ol.cross_entropy2d(ref_aux, y, 255)
    ref_loss.backward()
    m.train()
    crit = seg_b200.CrossEntropyLoss2d(ignore_index=255)
    yd = y.cuda()
    out = m(x.cuda())
    if kind == "pspnet":
        out, aux = out
        loss = crit(out, yd) + 0.4 * crit(aux, yd)
    else:
        loss = crit(out, yd)
    loss.backward()
    torch.cuda.synchronize()
    tag = f"[batch-stat {kind}/{backbone}{kw}]"
    log(gpu_out_dir, f"{tag} logits rel_err vs fp32 oracle {relerr(out, ref_out):.3e} (chaotic regime, see module docstring); "
                     f"loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert abs(loss.item() - ref_loss.item()) < 0.05 * abs(ref_loss.item())
    argmax_report(gpu_out_dir, tag, out, ref_out.detach())
    cos = []
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        cos.append(cosine(p.grad, osd[name].grad))
    cos_t = torch.tensor(cos)
    log(gpu_out_dir, f"{tag} grad cosine vs fp32 oracle (chaotic regime, informational): median {cos_t.median():.4f}, min {cos_t.min():.4f}")
    # early layers are upstream of little chaos: the stem's running statistics must match tightly
    esd = m.state_dict()
    stem_bn = {"deeplab": "backbone.layer0.1", "pspnet": "initial.0.1", "upernet": "backbone.initial.1"}[kind]
    if backbone == "xception":
        stem_bn = "backbone.bn1"
    for k in (stem_bn + ".running_mean", stem_bn + ".running_var"):
        assert relerr(esd[k], osd[k]) < 1e-2, k
    rs = max(relerr(esd[k], osd[k]) for k in esd if k.endswith("running_mean") or k.endswith("running_var"))
    log(gpu_out_dir, f"{tag} BN running stats worst rel_err vs oracle {rs:.3e}")
    assert all(int(esd[k]) == 1 for k in esd if k.endswith("num_batches_tracked"))


def test_batchstat_train_step_shallow_trunk(gpu_out_dir):
    """Batch-statistics BN forward+backward IN CONTEXT on a network shallow enough (Bottleneck blocks 1-1-1-1, same code
    path as resnet50/101) that rounding noise is not amplified into chaos: tight comparison with the fp32 oracle."""
    nc, backbone, kw = 19, "resnet14", dict(output_stride=16)
    sd, m = build("deeplab", nc, backbone, 6, **kw)
    x, y = synth.make_batch(4, 129, 129, nc, 255, seed=9003)
    osd = om.clone_sd(sd, requires_grad=True)
    ref_out = om.deeplab_forward(osd, x, backbone=backbone, train=True, **kw)
    ref_loss = ol.cross_entropy2d(ref_out, y, 255)
    ref_loss.backward()
    m.train()
    out = m(x.cuda())
    loss = seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    tag = "[batch-stat deeplab/resnet14]"
    e = relerr(out, ref_out)
    log(gpu_out_dir, f"{tag} logits rel_err vs fp32 oracle {e:.3e}; loss H100={loss.item():.6f} oracle={ref_loss.item():.6f}")
    assert e < 0.15 and abs(loss.item() - ref_loss.item()) < 1e-2 * abs(ref_loss.item())
    agree_all, agree_safe = argmax_report(gpu_out_dir, tag, out, ref_out.detach())
    assert agree_safe == 1.0 and agree_all > 0.9
    cos_min, cos_name = 1.0, None
    for name, p in m.named_parameters():
        c = cosine(p.grad, osd[name].grad)
        if c < cos_min:
            cos_min, cos_name = c, name
    log(gpu_out_dir, f"{tag} grads vs fp32 oracle: min cosine {cos_min:.5f} at {cos_name}")
    assert cos_min > 0.8
    esd = m.state_dict()
    rs = max(relerr(esd[k], osd[k]) for k in esd if k.endswith("running_mean") or k.endswith("running_var"))
    log(gpu_out_dir, f"{tag} BN running stats worst rel_err vs oracle {rs:.3e}")
    assert rs < 3e-2


def test_eval_forward_and_simt_tc_agree(gpu_out_dir):
    sd, m = build("deeplab", 19, "resnet50", 2, output_stride=16)
    x, _ = synth.make_batch(2, 129, 129, 19, 255, seed=9004)
    with torch.no_grad():
        ref = om.deeplab_forward(om.clone_sd(sd), x, backbone="resnet50", train=False, output_stride=16)
    m.eval()
    with torch.no_grad():
        out_tc = m(x.cuda())
        m.conv_impl = IMPL_SIMT
        out_simt = m(x.cuda())
    e1, e2, e3 = relerr(out_tc, ref), relerr(out_simt, ref), relerr(out_tc, out_simt)
    log(gpu_out_dir, f"[eval deeplab/r50] vs fp32 oracle: wgmma path {e1:.3e}; CUDA-core path {e2:.3e}; wgmma vs CUDA-core {e3:.3e} (bf16 noise floor)")
    assert e1 < 5e-2 and e2 < 5e-2 and e3 < 5e-2
    agree_all, agree_safe = argmax_report(gpu_out_dir, "[eval deeplab/r50]", out_tc, ref)
    assert agree_safe == 1.0 and agree_all > 0.97


def test_overfit_one_batch(gpu_out_dir):
    """Optimisation sanity: 40 fused train steps on one fixed batch must drive the loss down, as the oracle's SGD does."""
    sd, m = build("deeplab", 7, "resnet50", 4, output_stride=16)
    x, y = synth.make_batch(4, 65, 65, 7, 255, seed=9005)
    m.train()
    stepper = FusedTrainStep(m, ignore_index=255, lr=0.01, backbone_lr_scale=0.1, momentum=0.9, weight_decay=1e-4)
    xd, yd = x.cuda(), y.cuda()
    losses = [float(stepper.step(xd, yd).item()) for _ in range(40)]
    # oracle: same recipe on CPU, 12 steps (enough to see the same trend)
    osd = om.clone_sd(sd, requires_grad=True)
    names = om.param_names(osd)
    opt = torch.optim.SGD([{"params": [osd[n] for n in names if not n.startswith("backbone.")]},
                           {"params": [osd[n] for n in names if n.startswith("backbone.")], "lr": 0.001}], lr=0.01, momentum=0.9, weight_decay=1e-4)
    ref_losses = []
    for _ in range(12):
        opt.zero_grad()
        l = ol.cross_entropy2d(om.deeplab_forward(osd, x, backbone="resnet50", train=True), y, 255)
        l.backward()
        opt.step()
        ref_losses.append(l.item())
    log(gpu_out_dir, "[overfit] H100 fused-step loss: " + " ".join(f"{v:.3f}" for v in losses[:12]) + f" ... {losses[-1]:.3f}")
    log(gpu_out_dir, "[overfit] oracle SGD loss     : " + " ".join(f"{v:.3f}" for v in ref_losses))
    assert abs(losses[0] - ref_losses[0]) < 0.05 * ref_losses[0]
    assert losses[11] < 0.9 * losses[0] and ref_losses[11] < 0.9 * ref_losses[0]
    assert abs(losses[11] - ref_losses[11]) < 0.25 * ref_losses[11]
    assert losses[-1] < 0.6 * losses[0]
    assert all(v == v for v in losses)


def test_state_dict_keys_match_reference_inventory():
    m = seg_b200.DeepLab(19, backbone="resnet101")
    assert list(m.state_dict().keys()) == list(weights.deeplab_resnet_state_dict(19, "resnet101").keys())
    p = seg_b200.PSPNet(21, backbone="resnet50")
    assert list(p.state_dict().keys()) == list(weights.pspnet_state_dict(21, "resnet50").keys())
    xm = seg_b200.DeepLab(19, backbone="xception")
    assert list(xm.state_dict().keys()) == list(weights.deeplab_xception_state_dict(19).keys()) and xm._n_trainable() == 54704803
    u = seg_b200.UperNet(150, backbone="resnet101")
    assert list(u.state_dict().keys()) == list(weights.upernet_state_dict(150, "resnet101").keys())
    assert u._n_trainable() == 126414038
    assert p._n_trainable() == 51446762 and seg_b200.PSPNet(19, backbone="resnet50")._n_trainable() == 51444710
    assert len(list(m.get_backbone_params())) + len(list(m.get_decoder_params())) == len(list(m.parameters()))


def test_plugin_path_after_fused_steps_sees_updated_weights():
    """FusedTrainStep updates parameters in place (no autograd version bump) and keeps its own packed buffers; the
    autograd/plugin path used afterwards must repack the UPDATED weights and return a gradient for every parameter."""
    sd, m = build("deeplab", 7, "resnet14", 8, output_stride=16)
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9006)
    xd, yd = x.cuda(), y.cuda()
    m.train()
    with torch.no_grad():
        m.eval()
        before = m(xd).clone()
        m.train()
    st = FusedTrainStep(m, ignore_index=255, lr=0.05)
    for _ in range(2):
        st.step(xd, yd)
    m.eval()
    with torch.no_grad():
        after = m(xd)
    fresh = seg_b200.DeepLab(7, backbone="resnet14", output_stride=16).cuda()
    fresh.load_state_dict(m.state_dict())
    fresh.eval()
    with torch.no_grad():
        ref = fresh(xd)
    assert relerr(after, ref) < 1e-6, "plugin path used stale packed weights"
    assert relerr(after, before) > 1e-3, "the fused steps did not change the weights"
    m.train()
    out = m(xd)
    seg_b200.CrossEntropyLoss2d(ignore_index=255)(out, yd).backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())


@pytest.mark.parametrize("frozen_bn", [True, False], ids=["frozen-bn", "batch-stat"])
def test_graph_replayed_steps_equal_eager_steps(frozen_bn, gpu_out_dir):
    """CUDA-graph replay of the fused step (train.py: FusedTrainStep(cuda_graph=True)) is the same training as the eager
    step: the capture's two warm-up steps are rolled back, every replay is a fresh step (device-side counters).
    A second eager trainer is the control for run-to-run noise.  The BatchNorm statistics are accumulated exactly (fp64), so
    BOTH modes are reproducible: the three loss trajectories must agree to 1e-5 (fp32-atomic statistics made two EAGER
    batch-statistics runs differ by 1e-3) and the three-step parameter updates must be parallel (cosine > 0.9999)."""
    models = [build("deeplab", 7, "resnet14", 8, output_stride=16) for _ in range(3)]
    sd = models[0][0]
    m_e, m_c, m_g = (m for _, m in models)
    for m in (m_e, m_c, m_g):
        m.engine_dropout = False
        m.train()
        if frozen_bn:
            m.freeze_bn()
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9010)
    xd, yd = x.cuda(), y.cuda()
    lr = 1e-7 if frozen_bn else 0.005
    se, sc, sg = FusedTrainStep(m_e, lr=lr), FusedTrainStep(m_c, lr=lr), FusedTrainStep(m_g, lr=lr, cuda_graph=True)
    for i in range(3):
        le, lc, lg = float(se.step(xd, yd)), float(sc.step(xd, yd)), float(sg.step(xd, yd))
        noise = abs(le - lc) / abs(le)
        log(gpu_out_dir, f"graph-vs-eager [{'frozen-bn' if frozen_bn else 'batch-stat'}] step {i}: eager {le:.6f} control {lc:.6f} graph {lg:.6f}")
        assert le == le and abs(le - lg) <= 1e-5 * abs(le) and noise <= 1e-5, (i, le, lc, lg)
    assert sg.steps == 3
    upd = [torch.cat([(p.detach().cpu() - sd[n]).reshape(-1) for n, p in m.named_parameters()]) for m in (m_e, m_c, m_g)]
    c_ctrl, c_graph = cosine(upd[0], upd[1]), cosine(upd[0], upd[2])
    log(gpu_out_dir, f"graph-vs-eager [{'frozen-bn' if frozen_bn else 'batch-stat'}] 3 steps: update cosine {c_graph:.5f} (eager-vs-eager control {c_ctrl:.5f})")
    assert c_graph > 0.9999 and c_ctrl > 0.9999
    for (n, a), (_, b) in zip(m_e.named_buffers(), m_g.named_buffers()):
        if n.endswith("num_batches_tracked"):
            assert int(a) == int(b) == (0 if frozen_bn else 3), n


def test_training_step_is_bit_reproducible(gpu_out_dir):
    """Two trainers from the same state on the same batch, graph-replayed as bench.py runs them, must agree BIT FOR BIT after
    three steps: losses, the flat gradient of the last step, the parameters and the BatchNorm running statistics.  The shape
    is chosen so the paths whose sums could depend on arrival order all run: split-K weight gradients (few output tiles ->
    several k-splits, summed in split order) and the fused upsample + CE backward (overlapping bilinear footprints, summed in
    fixed point)."""
    models = [build("deeplab", 7, "resnet14", 8, output_stride=16) for _ in range(2)]
    for _, m in models:
        m.engine_dropout = False
        m.train()
    x, y = synth.make_batch(2, 65, 65, 7, 255, seed=9011)
    xd, yd = x.cuda(), y.cuda()
    steppers = [FusedTrainStep(m, lr=0.005, cuda_graph=True) for _, m in models]
    losses = [[float(s.step(xd, yd)) for _ in range(3)] for s in steppers]
    torch.cuda.synchronize()
    log(gpu_out_dir, f"bit-reproducibility: losses {losses[0]} / {losses[1]}")
    assert losses[0] == losses[1]
    assert torch.equal(steppers[0].flat_grad, steppers[1].flat_grad), "last step's gradients differ between identical runs"
    for (n, a), (_, b) in zip(models[0][1].named_parameters(), models[1][1].named_parameters()):
        assert torch.equal(a, b), n
    for (n, a), (_, b) in zip(models[0][1].named_buffers(), models[1][1].named_buffers()):
        assert torch.equal(a, b), n
