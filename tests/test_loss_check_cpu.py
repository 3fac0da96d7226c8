"""The loss checker (tests/loss_check.py) on the CPU: it accepts ATen's float32 results (F.cross_entropy,
oracle/losses_weighted.py and oracle.losses.lovasz_softmax through autograd, the last with its own sort of its own
rounded errors) and rejects planted defects of the kinds the kernels could have.  The defects are planted at the
largest pixel counts and class counts of the GPU sweep's per-element cases (for Lovász at a size the CPU sorts
quickly, with a rare class whose Jaccard steps are large, as in the sweep's largest case), where the bound is widest.

The Lovász bound is per element and does not widen with the pixel count: a member's allowance is the range of Jaccard
steps of its cluster of near-equal errors, and a step of a class with G foreground pixels after cb background ranks
is about G / (G + cb)^2.  A rare class (G = 3 here and in the sweep's 2^23 - 1 pixel case) has steps of 1/4, 3/20, ...
at its top ranks, far above the clusters' spread, so the shifted, sign-flipped and dropped classes are caught at any
pixel count; the tie defect is planted where tied groups rank at the top of the rare class, as in the sweep."""
import pytest
import torch
import torch.nn.functional as F

import loss_check as lc
from loss_check import labels, logits, lovasz_case, tie_case, weights
from oracle import losses as ol
from oracle import losses_weighted as olw

F32 = torch.float32


def aten_loss_grad(z, t, ignore, kind, w=None, gamma=0.0, mean=True, gscale=1.0):
    """ATen float32 loss and gradient through autograd."""
    zz = z.clone().requires_grad_(True)
    if kind == "focal":
        loss = olw.focal_loss(zz, t, gamma=gamma, alpha=w, ignore_index=ignore, size_average=mean)
    else:
        loss = olw.cross_entropy2d(zz, t, ignore_index=ignore, weight=w, reduction="mean" if mean else "sum")
    (loss * gscale).backward()
    return loss.detach(), zz.grad


# sizes: the sweep's largest per-element CE case is 3 * 132 * 8 * 256 + 17 pixels at C = 19
BIG = (1, 19, 811, 1000)


@pytest.mark.parametrize("kind,gamma,mean", [("ce", 0.0, True), ("wce", 0.0, True), ("wce", 0.0, False),
                                             ("focal", 0.0, True), ("focal", 0.5, True), ("focal", 2.0, False)])
def test_accepts_aten_fp32_loss_and_grad(kind, gamma, mean):
    N, C, H, W = 2, 21, 33, 37
    # ATen's focal autograd forms 0 * inf where pt rounds to 1 with gamma < 1 (oracle/losses_weighted.py): no saturation
    z = logits(N, C, H, W, 1, top=6 if gamma == 0 or gamma >= 1 else 0)
    # and wherever logpt = 0 (ignored pixels, zero-weight classes): neither of those either
    exact_aten = gamma == 0 or gamma >= 1
    t = labels(N, H, W, C, 2, frac=0.1 if exact_aten else 0.0)
    w = weights(C, 3) if kind != "ce" else None
    if w is not None and not exact_aten:
        w = w + 0.25
    loss, grad = aten_loss_grad(z, t, 255, kind, w, gamma, mean, gscale=0.75)
    r = lc.LossRef(z, t, 255, kind, w, gamma, mean)
    lc.check("aten", "dlogits", grad, r.grad_bound(0.75))
    r.check_loss("aten", loss)


def test_ce_reference_matches_oracle_float64():
    z = logits(2, 7, 9, 11, 4)
    t = labels(2, 9, 11, 7, 5)
    w = weights(7, 6)
    for kind, gamma in (("wce", None), ("focal", 0.5)):
        loss, grad = olw.weighted_loss_and_grad(z, t, 255, w, gamma, True)
        r = lc.LossRef(z, t, 255, kind, w, gamma or 0.0, True)
        assert abs(r.loss - float(loss)) <= 1e-12 * max(1.0, abs(float(loss)))
        assert torch.allclose(r.grad_bound().ref, grad, rtol=0, atol=1e-15)


def _big_case(kind, seed=7):
    N, C, H, W = BIG
    z = logits(N, C, H, W, seed)
    t = labels(N, H, W, C, seed + 1)
    w = weights(C, seed + 2) if kind != "ce" else None
    return z, t, w


def test_rejects_gradient_at_ignored_pixel():
    z, t, _ = _big_case("ce")
    _, grad = aten_loss_grad(z, t, 255, "ce")
    n, h, w = (t == 255).nonzero()[-1].tolist()
    grad[n, 3, h, w] = 1e-30
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlogits", grad, lc.LossRef(z, t, 255, "ce").grad_bound())


def test_rejects_focal_denominator_over_valid_pixels_only():
    z, t, w = _big_case("focal")
    r = lc.LossRef(z, t, 255, "focal", w, 2.0, True)
    with pytest.raises(AssertionError, match="accum\\[1\\]"):
        r.check_accum("planted", torch.tensor([r.sum, float((t != 255).sum())], dtype=torch.float64))
    _, grad = aten_loss_grad(z, t, 255, "focal", w, 2.0)
    grad *= t.numel() / float((t != 255).sum())
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlogits", grad, r.grad_bound())


def test_rejects_weight_of_class_instead_of_target():
    z, t, w = _big_case("wce")
    r = lc.LossRef(z, t, 255, "wce", w, 0.0, True)
    sm = F.softmax(z.double(), 1)
    onehot = F.one_hot(t.clamp_max(18), 19).permute(0, 3, 1, 2).double()
    grad = (sm - onehot) * w.double().view(1, -1, 1, 1) * (t != 255).unsqueeze(1) * r.g
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlogits", grad.float(), r.grad_bound())


def test_rejects_last_maximum_on_ties():
    z = logits(1, 150, 64, 64, 8)
    z[0, 5] = z[0, 77] = z.amax(1)[0] + 1  # every pixel ties classes 5 and 77
    t = labels(1, 64, 64, 150, 9)
    ref = lc.metrics_ref(z, t, 150)
    zf = z.flip(1)
    last = 149 - lc.first_argmax(zf)
    assert bool((last == 77).all()) and bool((lc.first_argmax(z) == 5).all())
    got = ref.clone()
    lab = (t >= 0) & (t < 150)
    got[2 + 150 + 5] -= int(lab.sum())
    got[2 + 150 + 77] += int(lab.sum())
    with pytest.raises(AssertionError, match="differ"):
        lc.check_exact("planted", "counters", got, ref, ("i",))


# ------------------------------------------------------------------------------------------------ Lovász
def lovasz_emulate(z, t, ignore, defect=None, cls=None):
    """float32 emulation of seg_lovasz.cu: keys sorted by (error descending, pixel ascending), Jaccard steps in fp32,
    the softmax Jacobian in fp32.  defect: None, 'shift' (class cls's d taken one rank down), 'sign' (class cls's
    fg/bg sign flipped), 'absent' (class cls treated as absent), 'ties' (tied errors ranked in reverse pixel order)."""
    N, C, H, W = z.shape
    p = F.softmax(z, 1).permute(0, 2, 3, 1).reshape(-1, C)
    lab = t.reshape(-1)
    valid = (lab != ignore).nonzero().flatten()
    pv, lv = p[valid], lab[valid]
    P = valid.numel()
    present = [c for c in range(C) if bool((lv == c).any()) and not (defect == "absent" and c == cls)]
    g = torch.zeros(P, C)
    loss = 0.0
    for c in present:
        fg = (lv == c).float()
        e = (fg - pv[:, c]).abs()
        pix = torch.arange(P)
        if defect == "ties":
            pix = P - 1 - pix
        o1 = torch.sort(pix, stable=True).indices
        order = o1[torch.sort(e[o1], descending=True, stable=True).indices]
        fs = fg[order]
        Gc = fs.sum()
        cf = torch.cumsum(fs, 0)
        cb = torch.arange(1, P + 1, dtype=F32) - cf
        j = 1 - (Gc - cf) / (Gc + cb)
        d = torch.cat([j[:1], j[1:] - j[:-1]])
        if defect == "shift" and c == cls:
            d = torch.cat([d[1:], d[-1:]])
        s = torch.where(fs > 0, -d, d)
        if defect == "sign" and c == cls:
            s = -s
        g[order, c] = s
        loss += float((e[order].double() * d.double()).sum())
    n = len(present)
    dot = (pv * g).sum(1, keepdim=True)
    dl = pv * (g - dot) / n
    full = torch.zeros(N * H * W, C)
    full[valid] = dl
    return loss / n, full.view(N, H, W, C).permute(0, 3, 1, 2)


def test_accepts_aten_fp32_lovasz():
    for C, seed in ((7, 21), (19, 22)):
        z = logits(2, C, 29, 31, seed, sat=True)
        t = labels(2, 29, 31, C, seed + 1)
        zz = z.clone().requires_grad_(True)
        loss = ol.lovasz_softmax(zz, t, 255)
        (loss * 1.0).backward()
        r = lc.LovaszRef(z, t, 255)
        lc.check("aten lovasz", "dlogits", zz.grad, r.grad)
        r.check_loss("aten lovasz", loss)


def test_accepts_emulation_with_tie_order():
    z, t = lovasz_case()
    loss, grad = lovasz_emulate(z, t, 255)
    r = lc.LovaszRef(z, t, 255, tie_order=True)
    lc.check("emulated lovasz", "dlogits", grad, r.grad)
    r.check_loss("emulated lovasz", loss)


@pytest.mark.parametrize("defect", ["shift", "sign", "absent"])
def test_rejects_lovasz_defects(defect):
    z, t = lovasz_case()
    r = lc.LovaszRef(z, t, 255)
    _, grad = lovasz_emulate(z, t, 255, defect, cls=0)
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlogits", grad, r.grad)


def test_rejects_ties_out_of_pixel_order():
    z, t = tie_case()
    r = lc.LovaszRef(z, t, 255, tie_order=True)
    assert r.pure_tie_clusters > 100
    _, grad = lovasz_emulate(z, t, 255)
    lc.check("ties in order", "dlogits", grad, r.grad)
    _, bad = lovasz_emulate(z, t, 255, "ties")
    lc.check("ties reversed, cluster tolerance", "dlogits", bad, lc.LovaszRef(z, t, 255).grad)
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlogits", bad, r.grad)


def test_schedule_mirrors():
    b, it, capped = lc.nchw_grid(3 * 132 * 8 * 256 + 17, 132)
    assert (b, it, capped) == (1056, 4, True)
    s = lc.lovasz_schedule(2 ** 23 - 1, 2 ** 23 - 1, 8, 132)
    assert s["nblocks"] > 1024 and s["radix_per"] == 8 and s["tiles"] == 2048 and s["class_scan_per"] == 2


# ------------------------------------------------------------------------------------------------ fused upsample / shuffle
def upsample_case(Hi=129, Ho=513, C=19, ac=1, seed=41):
    """The sweep's largest upsample shape (129 -> 513, align_corners, C = 19) in one image."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.randn(1, Hi, Hi, C, generator=g) * 3
    t = labels(1, Ho, Ho, C, seed + 1)
    return lo, t


def aten_upsample_grad(lo, t, ac):
    """ATen float32: F.interpolate + cross-entropy, autograd back to the NHWC low-res logits."""
    x = lo.clone().requires_grad_(True)
    up = F.interpolate(x.permute(0, 3, 1, 2), size=t.shape[1:], mode="bilinear", align_corners=bool(ac))
    loss = F.cross_entropy(up, t, ignore_index=255)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize("ac", [0, 1])
def test_accepts_aten_fp32_upsample(ac):
    lo, t = upsample_case(17, 65, 21, ac, 42)
    t = t[:, :65, :65]
    loss, grad = aten_upsample_grad(lo, t, ac)
    r = lc.UpsampleRef(lo, t, ac, 255, "ce")
    r.loss.check_loss("aten upsample", loss)
    lc.check("aten upsample", "dlo", grad, r.dlo_bound())


def test_rejects_dropped_output_pixel_and_wrong_lambda_row():
    lo, t = upsample_case()
    _, grad = aten_upsample_grad(lo, t, 1)
    r = lc.UpsampleRef(lo, t, 1, 255, "ce")
    b = r.dlo_bound()
    lc.check("aten upsample 129->513", "dlo", grad, b)
    gr, _ = r.grad_out()
    oy, ox = 300, 201
    drop = torch.einsum("h,c,w->hwc", r.Ay[oy], gr[0, :, oy, ox], r.Ax[ox]).unsqueeze(0)
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlo", grad - drop.float(), b)
    Ay_other = lc.lerp_matrix(129, 513, 0)
    Ay_bad = r.Ay.clone()
    Ay_bad[oy] = Ay_other[oy]
    wrong = lc.UpsampleRef.dlo_bound(r, Ay=Ay_bad).ref
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dlo", wrong.float(), b)


def shuffle_case(r=4, h=129, C=19, seed=51):
    """The sweep's largest shuffle case (r = 4, 129 x 129 low-res, C = 19) in one image; bf16 low-res logits."""
    g = torch.Generator().manual_seed(seed)
    lo = (torch.randn(1, h, h, r * r * C, generator=g) * 3).bfloat16()
    t = labels(1, h * r, h * r, C, seed + 1)
    return lo, t


def test_accepts_aten_shuffle_and_rejects_swapped_lanes_and_pad():
    r, C = 4, 19
    lo, t = shuffle_case(r, 129, C)
    x = lo.float().requires_grad_(True)
    F.cross_entropy(F.pixel_shuffle(x.permute(0, 3, 1, 2), r), t, ignore_index=255).backward()
    got = x.grad.bfloat16()
    ref = lc.ShuffleRef(lo, r, C, t, 255, "ce")
    b = ref.dx_bound()
    lc.check("aten shuffle", "dx", got, b)
    bad = got.clone()
    y, xx, c = 64, 77, 3
    bad[0, y, xx, c * r * r], bad[0, y, xx, c * r * r + 1] = got[0, y, xx, c * r * r + 1], got[0, y, xx, c * r * r]
    with pytest.raises(AssertionError, match="over the bound"):
        lc.check("planted", "dx", bad, b)
    padded = torch.zeros(1, 129, 129, r * r * C + 5, dtype=torch.bfloat16)
    padded[..., :r * r * C] = got
    lc.check_pad("shuffle pad", padded, r * r * C)
    padded[0, 5, 7, r * r * C + 2] = 1e-3
    with pytest.raises(AssertionError, match="pad lane"):
        lc.check_pad("planted", padded, r * r * C)


def test_fused_schedule_mirrors():
    s = lc.upsample_schedule(129, 129, 385, 385, 150, 1)
    assert s["fwd_ok"] and s["fwd_patch"] == 14 and s["bwd_tile"] == 16 and s["bwd_ok"]
    assert not lc.upsample_schedule(33, 33, 65, 65, 150, 0, metrics=False)["fwd_ok"]
    assert lc.upsample_schedule(129, 129, 513, 513, 19, 1)["last_tile_rows"] == 1
