"""Class-weighted cross-entropy and focal loss without a GPU: the float64 oracle against the values the reference's own
classes produced (tests/golden/losses_focal_weighted.npz, oracle/make_golden_losses.py), the bound on the focal gradient
factor that sizes the fused backward's fixed-point scale, and the argument checks of the engine's loss constructors."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import losses as ol
from oracle import losses_weighted as olw

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "losses_focal_weighted.npz")


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN)
    return g, json.loads(str(g["cases"]))


def _inputs(g, name):
    return (torch.from_numpy(g[f"in/{name}/logits"]), torch.from_numpy(g[f"in/{name}/target"]), int(g[f"in/{name}/ignore"]),
            torch.from_numpy(g[f"in/{name}/weight"]))


def _engine_def(g, case):
    logits, target, ign, w = _inputs(g, case["input"])
    weight = w.double() if case["weight"] else None
    mean = case["reduction"] == "mean"
    if case["kind"] == "ce_dice":
        ce, dce = olw.weighted_loss_and_grad(logits, target, ign, weight, None, mean)
        x = logits.double().clone().requires_grad_(True)
        dice = ol.dice_loss(x, target.clone())
        dice.backward()
        return ce + dice.detach(), dce + x.grad
    return olw.weighted_loss_and_grad(logits, target, ign, weight, case["gamma"], mean)


def test_golden_covers_the_cases(golden):
    g, cases = golden
    assert {c["input"].split("_")[0] for c in cases} == {"c19", "c21", "c150"}
    assert {c["gamma"] for c in cases if c["kind"] == "focal"} == {0.0, 0.5, 1.0, 2.0, 2.5}
    assert {c["reduction"] for c in cases} == {"mean", "sum"} and {c["weight"] for c in cases} == {False, True}
    for name in ("c19_img_ignored", "c19_all_ignored", "c19_zero_weight", "c19_saturated"):
        assert any(c["input"] == name for c in cases), name
    assert any(c["kind"] == "ce_dice" and c["weight"] for c in cases)
    assert int(g["in/c150/ignore"]) == -1
    w = g["in/c19/weight"]
    assert (w == 0).any() and (w > 0).any()


@pytest.mark.parametrize("kind", ["ce", "focal", "ce_dice"])
def test_oracle_matches_reference_golden(golden, kind):
    """loss to 1e-6 relative, gradients to 1e-5 of max|ref| where the reference's are finite.  Where they differ on purpose
    (DESIGN.md §4), the golden pins the reference's NaN and the oracle's finite value."""
    g, cases = golden
    n = 0
    for c in (c for c in cases if c["kind"] == kind):
        cid = c["id"]
        loss, grad = _engine_def(g, c)
        ref_l = float(g[f"{cid}/loss"])
        ref_g = torch.from_numpy(g[f"{cid}/grad"]).double()
        if math.isnan(ref_l):  # ATen's mean over a zero denominator; the engine defines it as 0 with gradient 0
            assert c["reduction"] == "mean" and kind == "ce", cid
            assert float(loss) == 0.0 and float(grad.abs().max()) == 0.0, cid
        else:
            assert abs(float(loss) - ref_l) <= 1e-6 * max(abs(ref_l), 1e-30), (cid, float(loss), ref_l)
        fin = torch.isfinite(ref_g)
        if fin.any():
            scale = float(ref_g[fin].abs().max())
            err = float((grad[fin] - ref_g[fin]).abs().max())
            assert err <= 1e-5 * max(scale, 1e-30), (cid, err, scale)
        assert torch.isfinite(grad).all(), cid
        if kind == "ce_dice":
            t = torch.from_numpy(g[f"{cid}/target_after"])
            t0 = torch.from_numpy(g[f"in/{c['input']}/target"])
            ol.dice_loss(torch.from_numpy(g[f"in/{c['input']}/logits"]), t0)  # mutates t0 like the reference
            assert torch.equal(t0, t), cid
        n += 1
    assert n > 0


def test_golden_pins_the_deliberate_differences(golden):
    g, _ = golden
    # FocalLoss, 0 < gamma < 1, pixels where pt rounds to 1: the reference's autograd gives NaN, the engine the limit
    cid = "c19_saturated/focal/now/mean/g0.5"
    ref = torch.from_numpy(g[f"{cid}/grad"])
    assert torch.isnan(ref[:, :, 1:3, :]).any() and torch.isfinite(ref[:, :, 3:, :]).all()
    _, grad = olw.weighted_loss_and_grad(*_inputs(g, "c19_saturated")[:3], None, 0.5, True)
    assert torch.isfinite(grad).all() and float(grad[:, :, 1:3, :].abs().max()) < 1e-30
    # the reference's one-pixel NaN case, in float32 autograd
    z = torch.tensor([[[[100.0]], [[0.0]], [[0.0]]]], requires_grad=True)
    olw.focal_loss(z, torch.zeros(1, 1, 1, dtype=torch.long), gamma=0.5).backward()
    assert torch.isnan(z.grad).any()
    # weighted mean over a zero denominator: NaN in ATen, 0 in the engine
    for cid in ("c19_all_ignored/ce/now/mean", "c19_all_ignored/ce/w/mean", "c19_zero_weight/ce/w/mean"):
        assert math.isnan(float(g[f"{cid}/loss"])), cid
    assert float(g["c19_all_ignored/focal/now/mean/g2.0/loss"]) == 0.0  # focal divides by every pixel: no NaN
    # CE_DiceLoss with ignored pixels: the reference cannot back-propagate (Dice rewrites the target CE saved)
    assert "backward_error" in "".join(g.files) and str(g["c19/ce_dice/now/mean/backward_error"])


def test_focal_grad_factor_bound_and_stable_form():
    """0 <= F'(L) <= 1 + gamma over L in [0, 100], gamma in [0, 4], and the stable form equals the textbook
    (1-pt)^g + g (1-pt)^(g-1) pt L wherever the latter is finite."""
    L = torch.cat([torch.zeros(1), torch.logspace(-30, 2, 4000, dtype=torch.float64), torch.linspace(0, 100, 4001, dtype=torch.float64)])
    for gamma in torch.linspace(0, 4, 81, dtype=torch.float64).tolist():
        f = olw.focal_grad_factor(L, gamma)
        assert torch.isfinite(f).all(), gamma
        assert float(f.min()) >= 0.0 and float(f.max()) <= 1.0 + gamma + 1e-12, gamma
        pt = torch.exp(-L)
        with np.errstate(all="ignore"):
            naive = (1 - pt) ** gamma + gamma * (1 - pt) ** (gamma - 1) * pt * L
        ok = torch.isfinite(naive) & (L > 1e-6)  # (1 - pt) cancels catastrophically below that
        assert torch.allclose(f[ok], naive[ok], rtol=1e-9, atol=1e-12), gamma
        # the derivative of F(L) = u^gamma L by central differences
        Lm = torch.linspace(0.01, 50, 500, dtype=torch.float64)
        h = 1e-6
        F = lambda x: (-torch.expm1(-x)) ** gamma * x  # noqa: E731
        assert torch.allclose(olw.focal_grad_factor(Lm, gamma), (F(Lm + h) - F(Lm - h)) / (2 * h), rtol=1e-5, atol=1e-8), gamma
    # the limit at L = 0: 1 for gamma = 0, 0 for gamma > 0
    assert float(olw.focal_grad_factor(torch.zeros(1, dtype=torch.float64), 0.0)) == 1.0
    assert float(olw.focal_grad_factor(torch.zeros(1, dtype=torch.float64), 0.5)) == 0.0


def test_oracle_focal_gamma0_is_ce_sum_over_all_pixels(golden):
    g, _ = golden
    logits, target, ign, _ = _inputs(g, "c19")
    focal, _ = olw.weighted_loss_and_grad(logits, target, ign, None, 0.0, True)
    ce_sum = olw.cross_entropy2d(logits.double(), target, ign, reduction="sum")
    assert abs(float(focal) - float(ce_sum) / target.numel()) <= 1e-12 * abs(float(focal))


def test_constructors_reject_bad_arguments():
    from seg_b200 import losses
    for bad in ([1.0, -0.5, 2.0], [1.0, float("nan")], [float("inf"), 1.0], [[1.0, 2.0]], []):
        with pytest.raises(ValueError):
            losses.CrossEntropyLoss2d(weight=bad)
        with pytest.raises(ValueError):
            losses.CE_DiceLoss(weight=bad)
        with pytest.raises(ValueError):
            losses.FocalLoss(alpha=bad)
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            losses.FocalLoss(gamma=bad)
    with pytest.raises(NotImplementedError):
        losses.CrossEntropyLoss2d(reduction="none")
    with pytest.raises(NotImplementedError):
        losses.CE_DiceLoss(reduction="none")
    with pytest.raises(ValueError):
        losses.CrossEntropyLoss2d(reduction="average")
    # accepted: sequences and 1-D tensors, zeros included; the length is checked against C at forward
    ce = losses.CrossEntropyLoss2d(weight=torch.tensor([0.0, 1.0, 2.5]), reduction="sum")
    assert ce.spec is not None and not ce.spec.mean and ce.spec.gamma is None
    with pytest.raises(ValueError):
        ce.spec.weight_on("cpu", 4)
    assert _is_plain_ce(losses.CrossEntropyLoss2d().spec)  # unweighted mean CE keeps the dedicated kernels
    f = losses.FocalLoss()
    assert f.spec.gamma == 2.0 and f.spec.mean and f.spec.weight is None and f.ignore_index == 255


def _is_plain_ce(spec):
    """spec is the unweighted mean cross-entropy, and the ops layer runs it on the SEG_LOSS_CE kernels."""
    from seg_b200 import lib, ops
    return (spec.weight is None and spec.mean and spec.gamma is None
            and ops._loss_kind(spec.weight, spec.gamma, spec.mean) == lib.LOSS_CE)


def test_specs_select_the_loss_kernels():
    from seg_b200 import lib, losses, ops
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "seg_b200.h")).read()
    for name in ("CE", "WCE", "FOCAL"):
        assert f"#define SEG_LOSS_{name} {getattr(lib, 'LOSS_' + name)}\n" in header, name
    kind = lambda crit: ops._loss_kind(crit.spec.weight, crit.spec.gamma, crit.spec.mean)  # noqa: E731
    assert kind(losses.CrossEntropyLoss2d()) == lib.LOSS_CE
    assert kind(losses.CrossEntropyLoss2d(reduction="sum")) == lib.LOSS_WCE
    assert kind(losses.CrossEntropyLoss2d(weight=[1.0, 2.0])) == lib.LOSS_WCE
    assert kind(losses.FocalLoss()) == lib.LOSS_FOCAL
    assert kind(losses.FocalLoss(gamma=0, alpha=[1.0, 2.0], size_average=False)) == lib.LOSS_FOCAL


def test_loss_entry_points_reject_bad_kinds():
    """The C ABI checks `kind` on the host before anything reaches the device (so no GPU is needed here): an unknown kind,
    SEG_LOSS_CE with a class weight or as a sum, and a negative focal gamma are errors."""
    from seg_b200 import lib
    so = lib.load()
    w = 256  # never dereferenced: the checks reject the call first
    nchw = (None, None, 1, 4, 1, 1, 255)
    up = (None, None, 1, 2, 2, 4, 4, 4, 0, 255)
    calls = [("unknown kind", so.seg_loss_nchw_fwd, nchw + (None, 3, 0.0, None, None)),
             ("unknown kind", so.seg_upsample_loss_fwd, up + (None, -1, 0.0, None, None, None, None)),
             ("SEG_LOSS_CE", so.seg_loss_nchw_fwd, nchw + (w, lib.LOSS_CE, 0.0, None, None)),
             ("SEG_LOSS_CE", so.seg_loss_nchw_bwd, nchw + (None, lib.LOSS_CE, 0.0, 0, None, None, None, None)),
             ("SEG_LOSS_CE", so.seg_upsample_loss_bwd, up + (w, lib.LOSS_CE, 0.0, 1, None, None, None, None, None, 8, None)),
             ("gamma", so.seg_upsample_loss_fwd, up + (None, lib.LOSS_FOCAL, -1.0, None, None, None, None))]
    for what, fn, args in calls:
        assert fn(*args) != 0, what
        assert what in lib.last_error(), (what, lib.last_error())


def test_fused_train_step_loss_argument_checks():
    from seg_b200 import losses
    from seg_b200.train import _loss_spec
    ii, spec = _loss_spec(None, None)
    assert ii == 255 and _is_plain_ce(spec)
    ii, spec = _loss_spec(None, 7)
    assert ii == 7 and _is_plain_ce(spec)
    ii, spec = _loss_spec(losses.FocalLoss(ignore_index=-1), None)
    assert ii == -1 and spec.gamma == 2.0
    assert _loss_spec(losses.CrossEntropyLoss2d(ignore_index=3), 3)[0] == 3
    with pytest.raises(ValueError):
        _loss_spec(losses.CrossEntropyLoss2d(ignore_index=3), 255)
    for crit in (losses.DiceLoss(), losses.CE_DiceLoss(), losses.LovaszSoftmax()):
        with pytest.raises(NotImplementedError, match="plugin surface"):
            _loss_spec(crit, None)


def test_registry_exports_focal_loss():
    import seg_b200
    from seg_b200 import losses
    assert seg_b200.FocalLoss is losses.FocalLoss
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorch-segmentation_b200",
                            "overlay", "utils", "losses.py")).read()
    assert "FocalLoss" in src.split("from seg_b200.losses import")[1].splitlines()[0]
