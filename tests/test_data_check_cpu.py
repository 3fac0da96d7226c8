"""The seg_data.cu checker (tests/data_check.py) on the CPU: it accepts correct results computed in another order (fp32
numpy transcriptions of each kernel with and without FMA, ATen's CPU F.interpolate, the fused-rotation transcription), and
it rejects seeded defects, naming the coordinate.  The write coverage of the augmentation kernels is emulated from
aug_grid, so an iteration slot the kernel skips shows up as unwritten sentinels."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import data_check as dc
from oracle import data as od
from oracle import inference as oi

SMS = 132
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
COORD = r"\((b|p|n|c|y)=\d+|\(p, y, x\)=\(\d+"
F32 = np.float32


# ------------------------------------------------------------------------------------------------ grid mirrors
def test_aug_grid_reaches_the_loops_the_sweep_relies_on():
    g = dc.aug_grid(8, 380, 380, 132)   # the shipped config
    assert (g.per_image, g.stride, g.outer, g.max_u) == (132, 33792, 2, 3)
    assert dc.aug_grid(8 * 132 + 1, 7, 9, 132).per_image == 1
    assert dc.aug_grid(65535, 1, 3, 132) == dc.AugGrid(1, 256, 1, 0, 1)
    assert dc.stream_grid(dc.grid_cap_elements(132), 132) == dc.StreamGrid(1056, 1, False)
    assert dc.stream_grid(dc.grid_cap_elements(132) + 1, 132) == dc.StreamGrid(1056, 2, True)


def test_tail_generalisation_equals_the_oracle_on_square_crops():
    rs = np.random.RandomState(1)
    for (h, w, crop) in ((33, 70, 48), (60, 20, 48), (100, 120, 48)):
        im = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        lb = rs.randint(-5, 300, (h, w)).astype(np.int32)
        y0, x0 = int(rs.randint(0, max(h, crop) - crop + 1)), int(rs.randint(0, max(w, crop) - crop + 1))
        for flip in (False, True):
            rx, ry = od.sample_tail(im, lb, crop, y0, x0, flip, MEAN, STD)
            x, y = dc.aug_reference("plain", [(im, lb, y0, x0, flip)], crop, crop, MEAN, STD)
            assert torch.equal(x[0], rx) and torch.equal(y[0], ry)


# ------------------------------------------------------------------------------------------------ augmentation emulation
def lut(mean, std, fault=None):
    """The kernel's per-block table: ((float)v / 255 - mean[c]) / std[c] in fp32."""
    m, s = list(mean), list(std)
    if fault == "swap_mean_std":
        m[1], s[1] = s[1], m[1]
    v = np.arange(256, dtype=F32) / F32(255)
    return np.stack([((v - F32(m[c])) / F32(s[c])).astype(F32) for c in range(3)])


def emu_plain(sample, ch, cw, fault=None):
    """numpy transcription of augment_u8_kernel for one image: (uint8 [ch, cw, 3], int64 [ch, cw])."""
    img, lbl, y0, x0, flip = sample
    h, w = img.shape[:2]
    y, x = np.meshgrid(np.arange(ch), np.arange(cw), indexing="ij")
    if flip and fault == "flip_before_crop":   # mirrored within the padded image, then cropped
        sy, sx = y + y0, max(w, cw) - 1 - (x + x0)
    else:
        xs = ((ch if fault == "flip_crop_h" else cw) - 1 - x) if flip else x
        sy, sx = y + y0, xs + x0
    inside = ((sy <= h) & (sx <= w)) if fault == "pad_le" else ((sy < h) & (sx < w))
    # what lies past the image in the arena (the next sample's bytes): anything but the zero padding
    big = np.full((h + 1, w + 1, 3), 77, np.uint8)
    big[:h, :w] = img
    bl = np.full((h + 1, w + 1), 77, np.int64)
    if lbl is not None:
        bl[:h, :w] = lbl
    syc, sxc = np.clip(sy, 0, h), np.clip(sx, -w - 1, w)
    u8 = np.where(inside[..., None], big[syc, sxc], 0).astype(np.uint8)
    lab = np.where(inside, bl[syc, sxc], 0) if lbl is not None else np.zeros((ch, cw), np.int64)
    return u8, lab.astype(np.int64)


def emu_batch(kind, samples, ch, cw, mean=MEAN, std=STD, sms=SMS, fault=None, labels=True):
    """All B images of one launch into sentinel buffers, the elements written as the grid of aug_grid writes them."""
    B = len(samples)
    xg = dc.FlatGuarded((B, 3, ch, cw), torch.float32)
    lg = dc.FlatGuarded((B, ch, cw), torch.int64) if labels else None
    plane = ch * cw
    g = dc.aug_grid(B, ch, cw, sms)
    i = np.arange(plane)
    written = np.ones(plane, bool)
    if fault == "skip_u3":
        written = (i // g.stride) % dc.AUG_U != 3
    table = lut(mean, std, fault)
    xflat = xg.buf[xg.lead:xg.lead + xg.n]
    for b, s in enumerate(samples):
        if kind == "plain":
            u8, lab = emu_plain(s, ch, cw, fault)
            xb = torch.from_numpy(np.stack([table[c][u8[..., c]] for c in range(3)]))
        else:
            im, lb, h, w = s[:4]
            angle, (y0, x0, flip) = (None, s[4:]) if kind == "scale" else (s[4], s[5:])
            xb, labt = dc.fused_emulation(im, lb, h, w, angle, (ch, cw), y0, x0, bool(flip), mean, std, fault=fault)
            lab = labt.numpy()
        off = b * plane * (1 if (fault == "plane_offset" and b > 0) else 3)
        xb = xb.reshape(3, plane)
        for c in range(3):
            dst = xflat[off + c * plane:off + (c + 1) * plane]
            dst[torch.from_numpy(written)] = xb[c][torch.from_numpy(written)]
        if lg is not None:
            lv = lg.view[b].reshape(-1)
            lv[torch.from_numpy(written)] = torch.from_numpy(lab.reshape(-1))[torch.from_numpy(written)]
    return xg, lg


def run_check(kind, samples, ch, cw, xg, lg, mean=MEAN, std=STD):
    case = f"{kind} B={len(samples)} crop={ch}x{cw}"
    dc.check_guards(case, xg.buf, xg.guard_mask())
    dc.check_written(case, xg.view)
    if lg is not None:
        dc.check_guards(case, lg.buf, lg.guard_mask())
        dc.check_written(case, lg.view)
    xr, lr = dc.aug_reference(kind, samples, ch, cw, mean, std, want_labels=lg is not None)
    dc.check_augment(case, xg.view, None if lg is None else lg.view, xr, lr)


def make_samples(kind, n, ch, cw, seed, label_kinds=("u8", "i32"), src=(20, 70), angles=(-10, 7, 45, 90)):
    rs = np.random.RandomState(seed)
    out = []
    for k in range(n):
        H, W = int(rs.randint(*src)), int(rs.randint(*src))
        im = rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
        lk = label_kinds[k % len(label_kinds)]
        if lk == "u8":
            lb = rs.randint(0, 256, (H, W)).astype(np.uint8)
        elif lk == "i32":
            lb = rs.choice(np.array([-1, 255, 2**31 - 1, -2**31, 0, 7], np.int64), (H, W)).astype(np.int32)
        else:
            lb = None
        if kind == "plain":
            h, w = H, W
        else:
            h, w = int(rs.randint(10, 90)), int(rs.randint(10, 90))
        y0 = [0, max(h, ch) - ch, int(rs.randint(0, max(h, ch) - ch + 1))][k % 3]
        x0 = [max(w, cw) - cw, 0, int(rs.randint(0, max(w, cw) - cw + 1))][k % 3]
        flip = bool(k % 2)
        if kind == "plain":
            out.append((im, lb, y0, x0, flip))
        elif kind == "scale":
            out.append((im, lb, h, w, y0, x0, flip))
        else:
            out.append((im, lb, h, w, angles[k % len(angles)], y0, x0, flip))
    return out


GEOMS = [(4, 37, 53, 3), (3, 17, 60, 2), (3, 60, 17, 2), (5, 1, 1, 3), (9, 2, 5, 1), (4, 40, 60, 1)]   # (B, crop_h, crop_w, sms)


@pytest.mark.parametrize("kind", ["plain", "scale", "full"])
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "B{}_{}x{}_sms{}".format(*g))
def test_checker_accepts_the_kernel_transcriptions(kind, geom):
    B, ch, cw, sms = geom
    samples = make_samples(kind, B, ch, cw, seed=ch * 7 + cw, label_kinds=("u8", "i32", None))
    xg, lg = emu_batch(kind, samples, ch, cw, sms=sms)
    run_check(kind, samples, ch, cw, xg, lg)
    xg, _ = emu_batch(kind, samples, ch, cw, sms=sms, labels=False)   # images only
    run_check(kind, samples, ch, cw, xg, None)


def test_coverage_emulation_reaches_u3_and_several_outer_iterations():
    g = dc.aug_grid(*GEOMS[-1])
    assert g.outer >= 2 and g.max_u == 3 and dc.aug_grid(*DEFECTS[5][2]).max_u == 3


DEFECTS = [
    ("flip_before_crop", "plain", (3, 20, 30, 2)),
    ("flip_crop_h", "plain", (3, 17, 30, 2)),
    ("pad_le", "plain", (3, 64, 64, 2)),
    ("swap_mean_std", "plain", (2, 9, 11, 2)),
    ("plane_offset", "plain", (3, 9, 11, 2)),
    ("skip_u3", "plain", (4, 40, 60, 1)),
    ("round_u8", "scale", (2, 21, 23, 2)),
    ("round_label", "scale", (2, 21, 23, 2)),
    ("label_delta_16", "full", (3, 31, 29, 2)),
]


@pytest.mark.parametrize("fault,kind,geom", DEFECTS, ids=[d[0] for d in DEFECTS])
def test_checker_rejects_seeded_augmentation_defects(fault, kind, geom):
    B, ch, cw, sms = geom
    samples = make_samples(kind, B, ch, cw, seed=5, label_kinds=("u8", "i32"), src=(40, 80) if fault != "round_label" else (9, 13),
                           angles=(-9, 45, 90))
    if fault == "pad_le":   # crops that reach past the image on both axes
        samples = [(s[0][:50, :50], None if s[1] is None else s[1][:50, :50], 0, 0, s[4]) for s in samples]
    xg, lg = emu_batch(kind, samples, ch, cw, sms=sms, fault=fault)
    with pytest.raises(AssertionError, match=COORD + "|never written"):
        run_check(kind, samples, ch, cw, xg, lg)


# ------------------------------------------------------------------------------------------------ resize_nchw emulation
def fma32(a, b, c):
    """fp32 fma: the exact product plus c, rounded once (float64 holds the product of two fp32 values exactly)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def emu_resize(src, Hd, Wd, mode, flip=False, alpha=1.0, beta=0.0, old=None, fma=False, fault=None):
    """numpy transcription of resize_nchw_kernel; src fp32 [P, Hs, Ws] -> fp32 [P, Hd, Wd]."""
    s = src.numpy().astype(F32)
    P, Hs, Ws = s.shape
    ox = np.arange(Wd)
    sxi = Wd - 1 - ox if flip else ox
    if mode == 2:
        zh = (Hs - 1) / (Hd - 1) if Hd > 1 else 1.0
        zw = (Ws - 1) / (Wd - 1) if Wd > 1 else 1.0
        cy, cx = np.arange(Hd) * zh, sxi * zw
        y0 = np.minimum(cy.astype(np.int64), Hs - 1)
        x0 = np.minimum(cx.astype(np.int64), Ws - 1)
        y1, x1 = np.where(y0 < Hs - 1, y0 + 1, y0), np.where(x0 < Ws - 1, x0 + 1, x0)
        ty, tx = (cy - y0)[:, None], (cx - x0)[None, :]
        sd = s.astype(np.float64)
        a, b = sd[:, y0][:, :, x0], sd[:, y0][:, :, x1]
        c, d = sd[:, y1][:, :, x0], sd[:, y1][:, :, x1]
        r = ((1.0 - ty) * ((1.0 - tx) * a + tx * b) + ty * ((1.0 - tx) * c + tx * d)).astype(F32)
        if fault != "no_fill":
            fill = (cy[:, None] > Hs - 1) | (cx[None, :] > Ws - 1)
            r = np.where(fill, F32(0), r)
    else:
        ac = (mode == 1) != (fault == "align_swap")
        iy0, iy1, ly1, ly0 = (t.numpy() for t in dc.lerp_axis(Hs, Hd, ac))
        ix0, ix1, lx1, lx0 = (t.numpy() for t in dc.lerp_axis(Ws, Wd, ac))
        ix0, ix1, lx1, lx0 = ix0[sxi], ix1[sxi], lx1[sxi], lx0[sxi]
        a, b = s[:, iy0][:, :, ix0], s[:, iy0][:, :, ix1]
        c, d = s[:, iy1][:, :, ix0], s[:, iy1][:, :, ix1]
        h1, h0, w1, w0 = ly1[:, None], ly0[:, None], lx1[None, :], lx0[None, :]
        if fma:
            i0 = fma32(np.broadcast_to(w0, a.shape), a, (w1 * b).astype(F32))
            i1 = fma32(np.broadcast_to(w0, c.shape), c, (w1 * d).astype(F32))
            r = fma32(np.broadcast_to(h0, i0.shape), i0, (h1 * i1).astype(F32))
        else:
            r = (h0 * ((w0 * a).astype(F32) + (w1 * b).astype(F32)).astype(F32)
                 + h1 * ((w0 * c).astype(F32) + (w1 * d).astype(F32)).astype(F32)).astype(F32)
    al, be = F32(alpha), F32(beta)
    if fault == "ignore_beta":
        be = F32(0)
    if fault == "alpha_after_beta":
        return torch.from_numpy(((be * old.numpy() + r) * al).astype(F32) if be != 0 else (al * r).astype(F32))
    v = (al * r).astype(F32)
    if be == 0:
        return torch.from_numpy(v)
    o = old.numpy().astype(F32)
    out = fma32(np.full_like(o, be), o, v) if fma else ((be * o).astype(F32) + v).astype(F32)
    return torch.from_numpy(out)


def planes(P, H, W, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(P, H, W, generator=g) * scale + scale).float()


RESIZE_SHAPES = [(29, 41, 44, 30), (29, 41, 13, 97), (1, 1, 5, 7), (6, 9, 1, 1), (48, 64, 84, 112), (11, 7, 3, 21)]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("fma", [False, True])
def test_checker_accepts_resize_transcriptions(mode, fma):
    for k, (Hs, Ws, Hd, Wd) in enumerate(RESIZE_SHAPES):
        src = planes(3, Hs, Ws, 10 + k)
        old = planes(3, Hd, Wd, 20 + k)
        for flip in (False, True):
            for alpha, beta in ((1.0, 0.0), (0.25, 1.0), (-0.5, 2.0)):
                got = emu_resize(src, Hd, Wd, mode, flip, alpha, beta, old, fma=fma)
                b = dc.resize_bound(src, Hd, Wd, mode, flip, alpha, beta, old)
                dc.check_resize(f"mode{mode} {Hs}x{Ws}->{Hd}x{Wd}", got, b)


def test_checker_accepts_aten_interpolate_and_nan_dst_overwrite():
    for k, (Hs, Ws, Hd, Wd) in enumerate(RESIZE_SHAPES):
        src = planes(2, Hs, Ws, 40 + k)
        for ac in (False, True):
            got = F.interpolate(src[None], size=(Hd, Wd), mode="bilinear", align_corners=ac)[0]
            dc.check_resize("aten", got, dc.resize_bound(src, Hd, Wd, int(ac)))
    nan = torch.full((2, 9, 7), math.nan)
    src = planes(2, 5, 6, 3)
    dc.check_resize("nan dst", emu_resize(src, 9, 7, 1, old=nan), dc.resize_bound(src, 9, 7, 1, old=nan))


def test_zoom_transcription_matches_scipy_and_pins_the_black_edge():
    saw_fill = False
    for (Hs, Ws, Hd, Wd) in ((48, 48, 84, 84), (64, 48, 112, 84), (37, 53, 9, 13), (5, 3, 15, 1), (1, 4, 3, 12)):
        src = planes(2, Hs, Ws, Hs + Wd, 4.0)
        saw_fill |= bool(dc.zoom_fill_mask(Hs, Ws, Hd, Wd).any())
        dc.check_resize("zoom", emu_resize(src, Hd, Wd, 2), dc.resize_bound(src, Hd, Wd, 2))
    assert saw_fill


RESIZE_DEFECTS = [("align_swap", 0, (29, 41, 44, 30), 1.0, 0.0), ("align_swap", 1, (29, 41, 44, 30), 1.0, 0.0),
                  ("no_fill", 2, (48, 48, 84, 84), 1.0, 0.0), ("ignore_beta", 1, (9, 11, 13, 17), 0.5, 1.0),
                  ("alpha_after_beta", 0, (9, 11, 13, 17), 0.5, 2.0), ("alpha_after_beta", 2, (9, 11, 13, 17), 0.5, 2.0)]


@pytest.mark.parametrize("fault,mode,shape,alpha,beta", RESIZE_DEFECTS, ids=[f"{d[0]}-mode{d[1]}" for d in RESIZE_DEFECTS])
def test_checker_rejects_seeded_resize_defects(fault, mode, shape, alpha, beta):
    Hs, Ws, Hd, Wd = shape
    src, old = planes(2, Hs, Ws, 1, 4.0), planes(2, Hd, Wd, 2)
    got = emu_resize(src, Hd, Wd, mode, False, alpha, beta, old, fault=fault)
    with pytest.raises(AssertionError, match=COORD):
        dc.check_resize(fault, got, dc.resize_bound(src, Hd, Wd, mode, False, alpha, beta, old))


# ------------------------------------------------------------------------------------------------ window_add, div
def emu_window_add(old, src, y0, x0, h, w, flip=False, alpha=1.0, fma=False, fault=None):
    out = old.clone().numpy()
    s = src.numpy()
    Ws = s.shape[2]
    if fault == "full_tile":
        h, w = min(s.shape[1], out.shape[1] - y0), min(Ws, out.shape[2] - x0)
    x = np.arange(w)
    xs = ((w if fault == "flip_over_w" else Ws) - 1 - x) if flip else x
    v = s[:, :h][:, :, xs]
    o = out[:, y0:y0 + h, x0:x0 + w]
    a = F32(alpha)
    out[:, y0:y0 + h, x0:x0 + w] = fma32(np.full_like(v, a), v, o) if fma else (o + (a * v).astype(F32)).astype(F32)
    return torch.from_numpy(out)


@pytest.mark.parametrize("fma", [False, True])
def test_checker_accepts_window_add(fma):
    src = planes(4, 20, 33, 7)
    for (y0, x0, h, w) in ((0, 0, 20, 33), (7, 11, 13, 20), (30, 27, 20, 33), (0, 27, 1, 33), (49, 0, 1, 1)):
        for flip in (False, True):
            old = planes(4, 50, 60, y0 + x0)
            got = emu_window_add(old, src, y0, x0, h, w, flip, 0.5, fma)
            dc.check_window_add("window", got, old, src, y0, x0, h, w, flip, 0.5)


@pytest.mark.parametrize("fault", ["full_tile", "flip_over_w"])
def test_checker_rejects_seeded_window_defects(fault):
    src, old = planes(2, 20, 33, 7), planes(2, 50, 60, 8)
    got = emu_window_add(old, src, 7, 11, 13, 20, True, 0.5, fault=fault)
    with pytest.raises(AssertionError, match=COORD):
        dc.check_window_add(fault, got, old, src, 7, 11, 13, 20, True, 0.5)


def test_div_is_exact_and_rejects_a_reciprocal_product():
    x = planes(3, 9, 13, 4)
    cnt = torch.randint(0, 5, (9, 13), generator=torch.Generator().manual_seed(1)).float()
    x[:, cnt == 0] = 0.0
    dc.check_div("div", x / cnt, x, cnt)
    with pytest.raises(AssertionError, match=r"\(p, y, x\)"):
        dc.check_div("recip", x * (1.0 / cnt), x, cnt)


# ------------------------------------------------------------------------------------------------ label map
def emu_argmax(scores, fault=None):
    """numpy transcription of argmax_nchw_kernel; fault "parent": the previous kernel (running v > best, NaN skipped,
    +inf wins); "last_max": v >= best."""
    s = scores.numpy()
    N, C = s.shape[:2]
    best, arg = s[:, 0].copy(), np.zeros(s[:, 0].shape, np.int64)
    bad = ~(best < np.inf)
    for c in range(1, C):
        v = s[:, c]
        bad |= ~(v < np.inf)
        take = (v >= best) if fault == "last_max" else (v > best)
        best, arg = np.where(take, v, best), np.where(take, c, arg)
    if fault != "parent":
        arg = np.where(bad, 0, arg)
    return torch.from_numpy(arg)


def label_columns():
    """[1, 5, 1, W] score columns: ties, +-0, -inf, NaN / +inf at the first, a middle and the last class, and one
    near-zero tie the float64 softmax cannot resolve."""
    inf, nan = math.inf, math.nan
    cols = [[1, 3, 3, 0, 2], [0.0, -0.0, -1, -2, -3], [-0.0, 0.0, -1, -2, -3], [-inf, -inf, -inf, -inf, -inf],
            [-inf, 1, -inf, 1, 0], [nan, 1, 2, 3, 4], [1, 2, nan, 3, 0], [1, 2, 3, 4, nan], [inf, 1, 2, 3, 4],
            [1, 2, inf, 3, 0], [1, 2, 3, 4, inf], [1, nan, 3, 0, 0], [nan, inf, nan, -inf, 0],
            [0.0, 1e-45, -1, -1, -1], [5, 5, 5, 5, 5], [-1, -2, -3, -4, 7]]
    return torch.tensor(cols, dtype=torch.float32).t().contiguous().reshape(1, 5, 1, len(cols))


def test_label_rule_against_the_softmax_reference():
    s = label_columns()
    assert dc.softmax_labels(s)[0, 0, 13].item() == 0 and dc.label_rule(s)[0, 0, 13].item() == 1
    assert dc.check_labels("columns", emu_argmax(s), s) == 1   # exactly the documented near-zero tie differs
    r = torch.randn(2, 7, 19, 23, generator=torch.Generator().manual_seed(5))
    r[:, 3] = r[:, 1]
    assert dc.check_labels("random", emu_argmax(r), r) == 0
    assert torch.equal(dc.softmax_labels(torch.tensor([1, math.nan, 3.0]).view(1, 3, 1, 1)).flatten(), torch.tensor([0]))


@pytest.mark.parametrize("fault", ["parent", "last_max"])
def test_checker_rejects_seeded_argmax_defects(fault):
    s = label_columns()
    with pytest.raises(AssertionError, match=r"\(b=0, y=0, x=\d+\)"):
        dc.check_labels(fault, emu_argmax(s, fault), s)


# ------------------------------------------------------------------------------------------------ TTA pipeline
def emu_multi_scale(model, image, scales, C, flip):
    """numpy transcription of seg_b200.inference.multi_scale_predict (kernels by their transcriptions above)."""
    _, _, H, W = image.shape
    total = torch.zeros(C, H, W)
    w = 1.0 / len(scales)
    for scale in scales:
        Hs, Ws = int(round(H * float(scale))), int(round(W * float(scale)))
        scaled = image[0] if (Hs, Ws) == (H, W) else emu_resize(image[0], Hs, Ws, 2)
        pred = model(scaled[None])[0]
        if flip:
            pred_f = model(emu_resize(scaled, Hs, Ws, 1, flip=True)[None])[0]
            total = emu_resize(pred, H, W, 1, alpha=0.5 * w, beta=1.0, old=total, fma=True)
            total = emu_resize(pred_f, H, W, 1, flip=True, alpha=0.5 * w, beta=1.0, old=total, fma=True)
        else:
            total = emu_resize(pred, H, W, 1, alpha=w, beta=1.0, old=total, fma=True)
    return total


def emu_sliding(model, image, C, flip, fault=None):
    """numpy transcription of seg_b200.inference.sliding_predict.  fault "parent": empty windows are not skipped and reach
    window_add, which refuses w = 0 as seg_window_add_nchw_f32 does; "clamped": empty windows moved back inside."""
    from seg_b200.inference import sliding_windows
    _, _, H, W = image.shape
    tile, wins = sliding_windows(H, W)
    total = torch.zeros(C, H, W)
    count = torch.zeros(H, W)
    for (y0, y1, x0, x1) in wins:
        if y1 <= y0 or x1 <= x0:
            if fault == "parent":
                raise RuntimeError("seg_window_add_nchw_f32 failed: window_add: window does not fit")
            if fault == "clamped":
                x0 = max(0, x1 - tile[1])
            else:
                continue
        img = image[0, :, y0:y1, x0:x1]
        padded = torch.zeros(3, max(tile[0], img.shape[1]), max(tile[1], img.shape[2]))
        padded[:, :img.shape[1], :img.shape[2]] = img
        pred = model(padded[None])[0]
        h, w = y1 - y0, x1 - x0
        if flip:
            pred_f = model(emu_resize(padded, padded.shape[1], padded.shape[2], 1, flip=True)[None])[0]
            total = emu_window_add(total, pred, y0, x0, h, w, alpha=0.5)
            total = emu_window_add(total, pred_f, y0, x0, h, w, flip=True, alpha=0.5)
        else:
            total = emu_window_add(total, pred, y0, x0, h, w)
        count[y0:y1, x0:x1] += 1
    return total / count


def tta_case(H, W, seed):
    return torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("shape", [(37, 53), (64, 48), (300, 20), (100, 30)])
def test_checker_accepts_the_tta_transcriptions(shape, flip):
    C = 5
    model = oi.toy_model(C, seed=3)
    img = tta_case(*shape, seed=shape[0])
    with torch.no_grad():
        got = emu_sliding(model, img, C, flip)
        ref, mag = dc.tta_reference("slide", model, img, C, flip)
        usage, acc = dc.check_tta(f"slide {shape}", got, ref, mag, dc.sliding_terms(*shape, flip))
        dc.check_tta_labels(f"slide {shape}", dc.label_rule(got[None])[0], ref, acc)
        scales = [1.0, 1.5] if shape[0] < 100 else [1.0]
        got = emu_multi_scale(model, img, scales, C, flip)
        ref, mag = dc.tta_reference("ms", model, img, C, flip, scales)
        usage, acc = dc.check_tta(f"ms {shape}", got, ref, mag, len(scales) * (2 if flip else 1))
        dc.check_tta_labels(f"ms {shape}", dc.label_rule(got[None])[0], ref, acc)


def test_portrait_sliding_window_reference_has_uncovered_pixels_and_the_parent_path_is_rejected():
    C = 5
    model = oi.toy_model(C, seed=3)
    img = tta_case(300, 20, 1)
    with torch.no_grad():
        ref, mag = dc.tta_reference("slide", model, img, C, False)
        assert int(torch.isnan(ref[0]).sum()) == 3600
        with pytest.raises(RuntimeError, match="window_add"):
            emu_sliding(model, img, C, False, fault="parent")
        got = emu_sliding(model, img, C, False, fault="clamped")
        with pytest.raises(AssertionError, match=r"NaN on one side only, first \(c, y, x\)"):
            dc.check_tta("clamped", got, ref, mag, dc.sliding_terms(300, 20, False))
        lab = dc.label_rule(emu_sliding(model, img, C, False)[None])[0]
        assert (lab[torch.isnan(ref[0])] == 0).all()
