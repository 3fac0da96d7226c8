"""Pixel accuracy / mIoU counters from the fused upsample + loss forward (seg_upsample_loss_fwd with counters), the training
metrics of FusedTrainStep(metrics=True) and its validation pass FusedTrainStep.evaluate, on the H100.

The reference for the counters is the plugin path bit for bit: seg_eval_metrics_nchw over the full-resolution logits
seg_bilinear_logits_fwd produces (itself pinned to the reference's utils/metrics.py by tests/test_ops_gpu.py)."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import synth, weights

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import seg_b200
    from seg_b200 import lib, losses, metrics, ops
    from seg_b200.train import FusedTrainStep

DEV = "cuda"
KINDS = ("ce", "wce", "focal")


def log(gpu_out_dir, msg):
    print(msg)
    with open(os.path.join(gpu_out_dir, "fused_metrics.txt"), "a") as f:
        f.write(msg + "\n")


def kind_args(kind, C):
    """(weight, gamma) of the upsample_loss_fwd call for `kind`."""
    if kind == "ce":
        return None, None
    g = torch.Generator().manual_seed(C)
    w = (torch.rand(C, generator=g) * 2 + 0.1).to(DEV)
    return (w, None) if kind == "wce" else (w, 2.0)


def fused_fwd(lo, t, ac, ign, kind, counters=None, want_argmax=False):
    w, gamma = kind_args(kind, lo.shape[-1])
    return ops.upsample_loss_fwd(lo, t, ac, ign, w, gamma, want_argmax=want_argmax, counters=counters)


def plugin_counters(lo, t, ac, C):
    """What the plugin path counts: eval_metrics_nchw over the materialised full-resolution logits."""
    full = ops.bilinear_logits_fwd(lo, t.shape[1], t.shape[2], ac)
    return ops.eval_metrics_nchw(full, t, C), full


def make_inputs(N, C, Hi, Wi, Ho, Wo, ign, special, seed):
    g = torch.Generator().manual_seed(seed)
    lo = torch.randn(N, Hi, Wi, C, generator=g) * 3
    t = torch.randint(0, C, (N, Ho, Wo), generator=g)
    t[:, :3, :] = ign
    if special == "out_of_range":  # labels >= C that are not the ignore value: neither labeled nor ignored by the loss
        t[:, 5:9, :] = C + 3
        t[:, 9:11, :] = C
    elif special == "all_ignored":
        t[:] = ign
    elif special == "image_unlabeled":  # one image without a labeled pixel
        t[1] = ign
        t[1, :, :4] = C + 1
    elif special == "ties":  # two channels with identical low-res logits, larger than every other: the lower index wins
        lo[:, :, :, 5] = lo[:, :, :, 2] = lo.abs().amax(-1) + 1.0
    elif special == "ignore_in_range":  # ignore_index inside [0, C): ignored by the loss, still labeled for the metrics
        t[:, 10:20, :] = ign
    return lo.contiguous().to(DEV), t.to(DEV)


SMALL = (2, 17, 19, 65, 73)
CASES = [(C, ign, ac, kind, "none", "small") for C in (7, 19, 21, 150) for ign in (255, -1) for ac in (True, False)
         for kind in KINDS]
CASES += [(19, 255, ac, kind, sp, "small") for sp in ("out_of_range", "all_ignored", "image_unlabeled", "ties")
          for ac in (True, False) for kind in KINDS]
CASES += [(19, 0, ac, kind, "ignore_in_range", "small") for ac in (True, False) for kind in KINDS]
CASES += [(19, 255, True, "ce", "none", "c3"), (19, 255, True, "focal", "none", "c3"), (150, -1, False, "ce", "none", "c5"),
          (150, -1, False, "wce", "none", "c5")]
SHAPES = {"small": SMALL, "c3": (16, 129, 129, 513, 513), "c5": (8, 128, 128, 512, 512)}


@pytest.mark.parametrize("C,ign,ac,kind,special,shape", CASES)
def test_fused_counters_equal_plugin_path(C, ign, ac, kind, special, shape, gpu_out_dir):
    N, Hi, Wi, Ho, Wo = SHAPES[shape]
    if special == "ignore_in_range":
        ign = 0
    lo, t = make_inputs(N, C, Hi, Wi, Ho, Wo, ign, special, seed=C * 7 + Hi)
    cnt = torch.zeros(2 + 3 * C, dtype=torch.int64, device=DEV)
    loss_m, acc_m, am = fused_fwd(lo, t, ac, ign, kind, counters=cnt, want_argmax=True)
    loss_p, acc_p, _ = fused_fwd(lo, t, ac, ign, kind)
    ref, _ = plugin_counters(lo, t, ac, C)
    tag = f"{shape} C={C} ign={ign} ac={ac} {kind} {special}"
    assert torch.equal(cnt, ref), tag
    # the metrics do not touch the loss: the fp32 loss is bit-identical and so is the denominator.  The fp64 loss sum
    # combines the blocks' partial sums with atomics in arrival order, so its last bits vary between any two launches,
    # with or without metrics (focal terms span more than the 29 bits that keep a sum of fp32 values exact in fp64)
    assert torch.equal(loss_m, loss_p) and float(acc_m[1]) == float(acc_p[1]), tag
    assert abs(float(acc_m[0]) - float(acc_p[0])) <= 1e-13 * abs(float(acc_p[0])), tag
    # the counters are added, not overwritten
    fused_fwd(lo, t, ac, ign, kind, counters=cnt)
    assert torch.equal(cnt, 2 * ref), tag
    if special == "ties":
        assert int((am == 5).sum()) == 0 and bool((am == 2).all()), tag
    if special == "all_ignored":
        assert int(cnt[1]) == 0, tag
    if special == "image_unlabeled":
        one, _ = plugin_counters(lo[:1].contiguous(), t[:1].contiguous(), ac, C)
        assert int(ref[1]) == int(one[1]), tag  # image 1 contributes nothing
    if special == "ignore_in_range":
        assert int(ref[2 + 2 * C]) > 0, tag  # label 0 == ignore_index is still counted as labeled
    log(gpu_out_dir, f"counters {tag}: equal to the plugin path; labeled {int(ref[1])}, correct {int(ref[0])}")


@pytest.mark.parametrize("C,ac,shape", [(19, True, "small"), (150, False, "small"), (19, True, "c3"), (150, False, "c5")])
def test_fused_argmax_against_aten(C, ac, shape, gpu_out_dir):
    """The fused arg-max may differ from F.interpolate(...).argmax(1) (what the reference computes) only where the float64
    top-2 margin is within the fp32 interpolation error of both."""
    N, Hi, Wi, Ho, Wo = SHAPES[shape]
    lo, t = make_inputs(N, C, Hi, Wi, Ho, Wo, 255, "none", seed=11 + C)
    # near-ties in the left half: channel 4 within ~1e-6 relative of a dominant channel 1
    g = torch.Generator(device=DEV).manual_seed(C)
    big = lo.abs().amax(-1)[:, :, : Wi // 2] + 1.0
    lo[:, :, : Wi // 2, 1] = big
    lo[:, :, : Wi // 2, 4] = big * (1 + (torch.rand(big.shape, device=DEV, generator=g) - 0.5) * 2e-6)
    _, _, am = fused_fwd(lo, t, ac, 255, "ce", want_argmax=True)
    nchw = lo.permute(0, 3, 1, 2).contiguous()
    aten = F.interpolate(nchw, size=(Ho, Wo), mode="bilinear", align_corners=ac).argmax(1)
    diff = am.long() != aten
    n = int(diff.sum())
    if n:
        z64 = F.interpolate(nchw.double(), size=(Ho, Wo), mode="bilinear", align_corners=ac)
        top2 = z64.topk(2, dim=1).values
        margin = (top2[:, 0] - top2[:, 1])[diff]
        # an fp32 interpolated value is off the float64 one by at most ~6 roundings of max|corner| plus the rounding of
        # the fp32 source coordinate (up to max(Hi, Wi) * 2^-24 in each lerp weight, times |corner difference| <= 2 max);
        # two values each that far off can swap
        err = (8 + 4 * max(Hi, Wi)) * 2.0 ** -24 * float(lo.abs().max())
        tol = 2 * err
        assert float(margin.max()) <= tol, (n, float(margin.max()), tol)
    log(gpu_out_dir, f"argmax vs ATen {shape} C={C} ac={ac}: {n} of {am.numel()} pixels differ, all within the fp32 margin")


# ---------------------------------------------------------------------------------------------- FusedTrainStep
def _model(kind, seed, C=7):
    if kind == "deeplab":
        sd = weights.deeplab_resnet_state_dict(C, "resnet14", seed=seed, randomize_bn=True)
        m = seg_b200.DeepLab(C, backbone="resnet14", pretrained=False, output_stride=16)
    elif kind == "pspnet":
        sd = weights.pspnet_state_dict(C, "resnet14", seed=seed, randomize_bn=True)
        m = seg_b200.PSPNet(C, backbone="resnet14", pretrained=False)
    else:
        sd = weights.upernet_state_dict(C, "resnet14", seed=seed, randomize_bn=True)
        m = seg_b200.UperNet(C, backbone="resnet14", pretrained=False)
    m.load_state_dict(sd, strict=True)
    m.engine_dropout = False
    return m.cuda().train()


def _batch(kind, seed, n=2):
    s = 64 if kind == "upernet" else 65
    x, y = synth.make_batch(n, s, s, 7, 255, seed=seed)
    return x.to(DEV), y.to(DEV)


def _state(step):
    m = step.model
    return ([p.detach().clone() for p in m.parameters()] + [b.detach().clone() for b in m.buffers()]
            + [step.flat_mom.clone(), step.flat_grad.clone()])


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize("graph", [False, True])
def test_step_metrics_do_not_change_training(graph):
    x, y = _batch("pspnet", 9101)
    steps = [FusedTrainStep(_model("pspnet", 31), lr=0.005, cuda_graph=graph, metrics=met) for met in (False, True)]
    for _ in range(3):
        losses_ = [float(s.step(x, y)) for s in steps]
        assert losses_[0] == losses_[1]
        assert _same(_state(steps[0]), _state(steps[1]))
    for s in steps:
        s.release_graph()


def test_step_metrics_add_no_launch():
    x, y = _batch("deeplab", 9102)
    counts = []
    for met in (False, True):
        s = FusedTrainStep(_model("deeplab", 32), lr=0.005, metrics=met)
        s.step(x, y)
        torch.cuda.synchronize()
        lib.reset_launch_count()
        s.step(x, y)
        counts.append(lib.launch_count())
    assert counts[0] == counts[1], counts


@pytest.mark.parametrize("kind", ["deeplab", "pspnet"])
def test_first_step_counters_equal_plugin_training_output(kind, gpu_out_dir):
    """The first step's counters are eval_metrics of the main head of the plugin surface's training-mode output."""
    x, y = _batch(kind, 9103)
    m = _model(kind, 33)
    out = m(x)
    out = out[0] if isinstance(out, tuple) else out
    ref = ops.eval_metrics_nchw(out.detach().contiguous(), y, 7)
    s = FusedTrainStep(_model(kind, 33), lr=0.005, metrics=True)
    s.step(x, y)
    assert torch.equal(s.seg_counters, ref), (s.seg_counters.tolist(), ref.tolist())
    got = s.seg_metrics()
    want = metrics.seg_metrics(ref.cpu().numpy(), 7)
    assert got["Pixel_Accuracy"] == want["Pixel_Accuracy"] and got["Mean_IoU"] == want["Mean_IoU"]
    log(gpu_out_dir, f"first-step metrics {kind}: {got['Pixel_Accuracy']} / {got['Mean_IoU']} equal to the plugin path")


def test_graph_counters_equal_eager_and_reset_in_replayed_loop():
    x, y = _batch("pspnet", 9104)
    x2, y2 = _batch("pspnet", 9105)
    se = FusedTrainStep(_model("pspnet", 34), lr=0.005, metrics=True)
    sg = FusedTrainStep(_model("pspnet", 34), lr=0.005, metrics=True, cuda_graph=True)
    hist = []
    for i, (xb, yb) in enumerate([(x, y), (x2, y2), (x, y), (x2, y2)]):
        if i == 2:
            se.reset_metrics()
            sg.reset_metrics()
        for s in (se, sg):
            s.step(xb, yb)
        assert torch.equal(se.seg_counters, sg.seg_counters), i
        hist.append(se.seg_counters.clone())
    assert int(hist[1][1]) == int(hist[0][1]) * 2  # same labeled pixels per batch (synth's layout): accumulated
    assert int(hist[2][1]) == int(hist[0][1])      # counted from zero after the reset
    assert se.seg_metrics() == sg.seg_metrics()
    sg.release_graph()


_SPEC = {"ce": lambda: None,
         "wce": lambda: losses.CrossEntropyLoss2d(weight=[0.5, 1.0, 2.0, 0.0, 1.5, 0.7, 1.1], ignore_index=255),
         "focal": lambda: losses.FocalLoss(ignore_index=255)}


@pytest.mark.parametrize("kind", ["deeplab", "pspnet", "upernet"])
@pytest.mark.parametrize("loss", ["ce", "wce", "focal"])
def test_evaluate_equals_plugin_eval(kind, loss, gpu_out_dir):
    x, y = _batch(kind, 9106)
    m = _model(kind, 35)
    s = FusedTrainStep(m, lr=0.005, metrics=True, loss=_SPEC[loss]())
    s.step(x, y)  # trained state, initialised step counter
    s.reset_metrics()
    before, ctr, n_steps = _state(s), m._step_ctr.clone(), s.steps
    v = s.evaluate(x, y)
    torch.cuda.synchronize()
    assert m.training and s.steps == n_steps and torch.equal(m._step_ctr, ctr) and _same(_state(s), before)
    # the plugin surface on the same model: model.eval()(x), the loss, eval_metrics
    m.eval()
    with torch.no_grad():
        out = m(x)
        crit = _SPEC[loss]() or losses.CrossEntropyLoss2d(ignore_index=255)
        ref_loss = float(crit(out, y))
        ref = ops.eval_metrics_nchw(out.contiguous(), y, 7)
    m.train()
    assert torch.equal(s.seg_counters, ref), (s.seg_counters.tolist(), ref.tolist())
    e = abs(float(v) - ref_loss) / abs(ref_loss)
    log(gpu_out_dir, f"evaluate {kind} {loss}: loss {float(v):.7f} plugin {ref_loss:.7f} (rel {e:.1e}), counters equal")
    assert e <= 1e-6 and int(ref[1]) > 0


def test_step_after_evaluate_is_unchanged():
    x, y = _batch("pspnet", 9107)
    a = FusedTrainStep(_model("pspnet", 36), lr=0.005, metrics=True)
    b = FusedTrainStep(_model("pspnet", 36), lr=0.005, metrics=True)
    la = [float(a.step(x, y))]
    lb = [float(b.step(x, y))]
    a.evaluate(x, y)
    a.reset_metrics()
    b.reset_metrics()
    la.append(float(a.step(x, y)))
    lb.append(float(b.step(x, y)))
    assert la == lb
    assert _same(_state(a), _state(b)) and torch.equal(a.seg_counters, b.seg_counters)


def test_evaluate_graph_equals_eager_with_smaller_last_batch(gpu_out_dir):
    x, y = _batch("pspnet", 9108, n=3)
    se = FusedTrainStep(_model("pspnet", 37), lr=0.005, metrics=True)
    sg = FusedTrainStep(_model("pspnet", 37), lr=0.005, metrics=True, cuda_graph=True)
    for s in (se, sg):
        s.step(x[:2], y[:2])
        s.reset_metrics()
    # full batch twice, a smaller last batch, and a third shape past the bound of captured shapes (eager)
    for xb, yb in [(x[:2], y[:2]), (x[:2], y[:2]), (x[2:], y[2:]), (x, y)]:
        le, lg = float(se.evaluate(xb, yb)), float(sg.evaluate(xb, yb))
        assert le == lg
        assert torch.equal(se.seg_counters, sg.seg_counters)
    assert len(sg._eval_graphs) == FusedTrainStep.EVAL_GRAPHS_MAX
    # the training step's graph is unaffected by the validation graphs
    assert float(se.step(x[:2], y[:2])) == float(sg.step(x[:2], y[:2]))
    assert _same(_state(se), _state(sg))
    log(gpu_out_dir, f"evaluate graph vs eager: equal; metrics {sg.seg_metrics()['Mean_IoU']}")
    sg.release_graph()


def test_metrics_require_opt_in():
    s = FusedTrainStep(_model("deeplab", 38), lr=0.005)
    assert s.seg_counters is None
    with pytest.raises(RuntimeError, match="metrics=True"):
        s.seg_metrics()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_metrics_and_validation_loss(tmp_path):
    """Under torchrun, seg_metrics() and the validation loss equal one GPU on the concatenated batch."""
    out = tmp_path / "dp_metrics.txt"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", "29617", os.path.join(root, "tests", "fused_metrics_dp_worker.py"), str(out)],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert out.read_text().strip().endswith("ok")
