"""Conformance sweep of seg_data.cu: the three augmentation kernels (bit-exact against oracle/data.py's restatement of the
reference pipeline) and the four inference kernels of test-time augmentation (per-element float64 bounds), plus the TTA
pipeline of seg_b200.inference against oracle/inference.py.  Bounds and references: tests/data_check.py.

Every launch writes through lib.call into guarded buffers (sentinel words before and after, the output itself starting
as the sentinel unless the kernel reads it), so an unwritten element or a stray write is caught; every case runs twice
and must be bit-identical.  Sizes come from the SM count at run time, and the sweep asserts the loops it reaches: an
augmentation case with two or more outer iterations and u = 3, one with one block per image, and streaming cases at
cap * 256 and cap * 256 + 1 elements (cap = 8 blocks per SM).  Each case appends its bound usage to
gpu_out_dir/data_conformance.txt."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import data_check as dc
from oracle import inference as oi

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import inference as di
    from seg_b200 import lib
    from seg_b200.data import _ENTRY, _FULL_ENTRY, _SCALE_ENTRY, DeviceBatcher, inverse_rotation

if torch.cuda.is_available():  # the fp32 stand-in network must not run its convolutions in TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

DEV = "cuda"
MEANS = [([0.485, 0.456, 0.406], [0.229, 0.224, 0.225]), ([0.5, 0.25, 0.0], [0.5, 2.0, 0.125])]
INT32_EXTREMES = np.array([-1, 255, 2**31 - 1, -2**31, 0, 19], np.int64)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cap():
    return dc.grid_cap_elements(sms())


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "data_conformance.txt"), "a")
    f.write(f"# {torch.cuda.get_device_name(0)} sms={sms()}\n")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


# ------------------------------------------------------------------------------------------------ augmentation
ENTRY = {"plain": ("seg_augment_batch_u8", lambda: _ENTRY), "scale": ("seg_augment_scale_batch_u8", lambda: _SCALE_ENTRY),
         "full": ("seg_augment_full_batch_u8", lambda: _FULL_ENTRY)}


def pack(kind, samples):
    """The arena (images and labels back to back, int32 labels 4-byte aligned) and the entry table, as DeviceBatcher
    packs them; a sample without a label gets lbl_off = -1."""
    dt = ENTRY[kind][1]()
    B = len(samples)
    chunks, off = [], 0
    table = np.zeros(B, dtype=dt)
    for b, s in enumerate(samples):
        img, lbl = np.ascontiguousarray(s[0], dtype=np.uint8), s[1]
        H, W = img.shape[:2]
        img_off = off
        chunks.append(img.reshape(-1))
        pad = (-img.size) % 4
        chunks.append(np.zeros(pad, np.uint8))
        off += img.size + pad
        lbl_off, lb = -1, 1
        if lbl is not None:
            lbl = np.ascontiguousarray(lbl)
            lb = lbl.dtype.itemsize
            lbl_off = off
            raw = lbl.reshape(-1).view(np.uint8)
            chunks.append(raw)
            pad = (-raw.size) % 4
            chunks.append(np.zeros(pad, np.uint8))
            off += raw.size + pad
        if kind == "plain":
            table[b] = (img_off, lbl_off, H, W, s[2], s[3], int(bool(s[4])), lb)
        elif kind == "scale":
            h, w = s[2], s[3]
            table[b] = (img_off, lbl_off, 1.0 / (w / W), 1.0 / (h / H), H, W, h, w, s[4], s[5], int(bool(s[6])), lb)
        else:
            h, w, angle = s[2], s[3], s[4]
            table[b] = (img_off, lbl_off, 1.0 / (w / W), 1.0 / (h / H)) + inverse_rotation(w, h, angle) + \
                (H, W, h, w, s[5], s[6], int(bool(s[7])), lb)
    arena = torch.from_numpy(np.concatenate(chunks + [np.zeros(8, np.uint8)])).to(DEV)
    return arena, torch.from_numpy(table.view(np.uint8).copy()).to(DEV)


def c3(v):
    return (ctypes.c_float * 3)(*[float(x) for x in v])


def launch_aug(kind, arena, table, B, ch, cw, mean, std, labels):
    xg = dc.FlatGuarded((B, 3, ch, cw), torch.float32, device=DEV)
    lg = dc.FlatGuarded((B, ch, cw), torch.int64, device=DEV) if labels else None
    lib.call(ENTRY[kind][0], lib.ptr(arena), lib.ptr(table), B, ch, cw, c3(mean), c3(std), lib.ptr(xg.view),
             None if lg is None else lib.ptr(lg.view))
    torch.cuda.synchronize()
    return xg, lg


def run_aug(log, case, kind, samples, ch, cw, mean_std=MEANS[0], labels=True, reference=None):
    """Two launches into fresh guarded buffers: guards intact, every element written, bit-identical, and bit-exact
    against the reference (reference: precomputed (x, labels) for samples that repeat)."""
    mean, std = mean_std
    B = len(samples)
    arena, table = pack(kind, samples)
    runs = []
    for _ in range(2):
        xg, lg = launch_aug(kind, arena, table, B, ch, cw, mean, std, labels)
        for g in (xg, lg):
            if g is not None:
                dc.check_guards(case, g.buf, g.guard_mask())
                dc.check_written(case, g.view)
        runs.append((xg.view.cpu(), None if lg is None else lg.view.cpu()))
    (x, y), (x2, y2) = runs
    assert torch.equal(bits(x), bits(x2)) and (y is None or torch.equal(y, y2)), f"{case}: not bit-reproducible"
    xr, yr = reference if reference is not None else dc.aug_reference(kind, samples, ch, cw, mean, std, labels)
    dc.check_augment(case, x, y, xr, yr)
    g = dc.aug_grid(B, ch, cw, sms())
    log(f"aug {kind} {case} B={B} crop={ch}x{cw} exact per_image={g.per_image} stride={g.stride} outer={g.outer} "
        f"max_u={g.max_u} iters={g.iters}")
    return g, x, y


def label_map(rs, H, W, kind):
    if kind == "u8":
        return rs.randint(0, 256, (H, W)).astype(np.uint8)
    if kind == "i32":
        return rs.choice(INT32_EXTREMES, (H, W)).astype(np.int32)
    return None


def samples_for(kind, n, ch, cw, seed, src=(40, 90), dst=None, angles=(-10, -3, 0, 5, 10, 45, -45, 90, 180),
                label_kinds=("u8", "i32")):
    """n samples cycling through the origins {0, max}, {max, 0}, random and through the label kinds; sources src, resized
    to dst (scale / full; a callable (rs, H, W) -> (h, w), default a random size around the source)."""
    rs = np.random.RandomState(seed)
    out = []
    for k in range(n):
        H, W = (int(rs.randint(*src)), int(rs.randint(*src))) if isinstance(src[0], int) else src[k % len(src)]
        im = rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
        lb = label_map(rs, H, W, label_kinds[k % len(label_kinds)])
        if kind == "plain":
            h, w = H, W
        elif dst is None:
            h, w = max(1, int(H * rs.uniform(0.5, 2.0))), max(1, int(W * rs.uniform(0.5, 2.0)))
        else:
            h, w = dst(rs, H, W, k)
        y0 = [0, max(h, ch) - ch, int(rs.randint(0, max(h, ch) - ch + 1))][k % 3]
        x0 = [max(w, cw) - cw, 0, int(rs.randint(0, max(w, cw) - cw + 1))][k % 3]
        flip = bool((k // 3) % 2)
        if kind == "plain":
            out.append((im, lb, y0, x0, flip))
        elif kind == "scale":
            out.append((im, lb, h, w, y0, x0, flip))
        else:
            out.append((im, lb, h, w, angles[k % len(angles)], y0, x0, flip))
    return out


KINDS = ["plain", "scale", "full"]


@pytest.mark.parametrize("kind", KINDS)
def test_aug_shipped_configs_and_large_crops(log, kind):
    for i, (B, crop, src) in enumerate(((8, 380, (300, 560)), (8, 480, (380, 640)), (2, 513, (400, 600)))):
        s = samples_for(kind, B, crop, crop, seed=10 + i, src=src,
                        dst=lambda rs, H, W, k: (int(rs.randint(crop // 2, 2 * crop)), int(rs.randint(crop // 2, 2 * crop))))
        run_aug(log, f"shipped-{i}", kind, s, crop, crop, MEANS[i % 2])


@pytest.mark.parametrize("kind", KINDS)
def test_aug_coverage_of_the_grid_stride_loops(log, kind):
    """A crop sized from the SM count so that, at B = 8, every thread walks at least two outer iterations and (plain
    kernel) reaches u = 3; and B = 8 SMs + 1 small crops, one block per image with a partial last iteration."""
    side = math.isqrt(6 * sms() * dc.THREADS) + 1
    g, _, _ = run_aug(log, "sm-sized", kind, samples_for(kind, 8, side, side, seed=20, src=(side // 2, side + 40)), side, side)
    assert g.outer >= 2 and g.max_u == 3 and g.iters >= 5, g
    B = 8 * sms() + 1
    g, _, _ = run_aug(log, "one-block-per-image", kind, samples_for(kind, B, 23, 31, seed=21, src=(5, 40)), 23, 31, MEANS[1])
    assert g.per_image == 1 and 0 < g.max_u < 3 and (23 * 31) % g.stride != 0, g


@pytest.mark.parametrize("kind", KINDS)
def test_aug_65535_images_at_a_1x3_crop(log, kind):
    base = samples_for(kind, 97, 1, 3, seed=30, src=(1, 6), dst=lambda rs, H, W, k: (int(rs.randint(1, 5)), int(rs.randint(1, 6))))
    xr, yr = dc.aug_reference(kind, base, 1, 3, *MEANS[0])
    idx = torch.arange(65535) % 97
    run_aug(log, "B65535", kind, [base[i] for i in idx.tolist()], 1, 3, reference=(xr[idx], yr[idx]))


@pytest.mark.parametrize("kind", KINDS)
def test_aug_geometry_edges(log, kind):
    cases = [("1x1", 1, 1, (1, 9)), ("17x300", 17, 300, (10, 400)), ("300x17", 300, 17, (10, 400)),
             ("crop-past-one-axis", 100, 100, [(50, 400), (400, 50)])]
    for name, ch, cw, src in cases:
        for j, (lk, ms) in enumerate(((("u8", "i32", None), MEANS[0]), (("i32",), MEANS[1]))):
            s = samples_for(kind, 6, ch, cw, seed=40 + j + ch, src=src, label_kinds=lk,
                            dst=None if name != "crop-past-one-axis" else (lambda rs, H, W, k: (H, W)))
            run_aug(log, f"{name}-{j}", kind, s, ch, cw, ms)
            run_aug(log, f"{name}-{j}-images-only", kind, s, ch, cw, ms, labels=False)


def test_aug_scale_extremes(log):
    """1-pixel sources, x8 and x1/8 ratios, exact x2 and x1/2."""
    dims = [lambda rs, H, W, k: (max(1, H * 8), max(1, W * 8)), lambda rs, H, W, k: (max(1, H // 8), max(1, W // 8)),
            lambda rs, H, W, k: (2 * H, 2 * W), lambda rs, H, W, k: (max(1, H // 2), max(1, W // 2)),
            lambda rs, H, W, k: (int(rs.randint(1, 40)), int(rs.randint(1, 40)))]
    for kind in ("scale", "full"):
        for i, dst in enumerate(dims):
            src = [(1, 1), (1, 50), (50, 1), (3, 5)] if i in (0, 4) else (16, 96)
            s = samples_for(kind, 8, 33, 41, seed=50 + i, src=src, dst=dst, angles=(0, 7, -10))
            run_aug(log, f"ratio-{i}", kind, s, 33, 41)


def test_aug_rotation_angles_and_angle_zero_equals_the_scale_kernel(log):
    angles = tuple(range(-10, 11)) + (45, -45, 90, -90, 180, -170)
    s = samples_for("full", len(angles), 64, 80, seed=60, src=(40, 120), angles=angles)
    run_aug(log, "angles", "full", s, 64, 80)
    zero = [t[:4] + (0,) + t[5:] for t in s]
    _, xf, yf = run_aug(log, "angle-0", "full", zero, 64, 80)
    _, xs, ys = run_aug(log, "angle-0-as-scale", "scale", [t[:4] + t[5:] for t in s], 64, 80)
    assert torch.equal(bits(xf), bits(xs)) and torch.equal(yf, ys), "angle 0 differs from the scale kernel"


def test_refusals_raise_before_any_launch():
    im = np.zeros((4, 5, 3), np.uint8)
    arena, table = pack("plain", [(im, None, 0, 0, False)] * 65536)
    out = torch.empty(65536 * 3 * 2, device=DEV)
    n0 = lib.launch_count()
    with pytest.raises(RuntimeError, match="bad batch"):
        lib.call("seg_augment_batch_u8", lib.ptr(arena), lib.ptr(table), 65536, 1, 2, c3(MEANS[0][0]), c3(MEANS[0][1]),
                 lib.ptr(out), None)
    b = DeviceBatcher(*MEANS[0], 8, DEV, max_bytes=1 << 20)
    bad = [[(im, None, -1, 0, False)], [(im, None, 0, 4, False)], [(im, None, 5, 0, False)]]
    for s in bad:
        with pytest.raises(ValueError, match="crop origin"):
            b.stage(s)
    with pytest.raises(ValueError, match="crop origin"):
        b.stage_scaled([(im, None, 20, 30, 0, 23, False)])
    with pytest.raises(ValueError, match="crop origin"):
        b.stage_full([(im, None, 20, 30, 5, -2, 0, False)])
    torch.cuda.synchronize()
    assert lib.launch_count() == n0, "a refused call launched a kernel"


# ------------------------------------------------------------------------------------------------ resize_nchw
def planes(P, H, W, seed, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(P, H, W, generator=g) + offset).float()


def run_resize(log, case, src, Hd, Wd, mode, flip=False, alpha=1.0, beta=0.0, old=None, nan_dst=False):
    P, Hs, Ws = src.shape
    b = dc.resize_bound(src, Hd, Wd, mode, flip, alpha, beta, old)
    s = src.contiguous().to(DEV)
    runs = []
    for _ in range(2):
        g = dc.FlatGuarded((P, Hd, Wd), torch.float32, device=DEV)
        if beta != 0.0:
            g.view.copy_(old)
        elif nan_dst:
            g.view.fill_(math.nan)
        lib.call("seg_resize_nchw_f32", lib.ptr(s), P, Hs, Ws, lib.ptr(g.view), Hd, Wd, mode, int(flip), float(alpha), float(beta))
        torch.cuda.synchronize()
        dc.check_guards(case, g.buf, g.guard_mask())
        dc.check_written(case, g.view)
        runs.append(g.view.cpu())
    assert torch.equal(bits(runs[0]), bits(runs[1])), f"{case}: not bit-reproducible"
    u = dc.check_resize(case, runs[0], b)
    sg = dc.stream_grid(P * Hd * Wd, sms())
    log(f"resize mode={mode} {case} {P}x{Hs}x{Ws}->{Hd}x{Wd} flip={int(flip)} alpha={alpha} beta={beta} usage={u:.4f} "
        f"blocks={sg.blocks} iters={sg.iters}")
    return u, runs[0]


SHAPES = [(6, 29, 41, 29, 41), (6, 29, 41, 44, 30), (6, 29, 41, 13, 97), (2, 1, 1, 5, 7), (3, 1, 9, 4, 1),
          (3, 6, 9, 1, 1), (2, 9, 1, 1, 12), (4, 48, 64, 84, 112), (2, 11, 7, 3, 21)]
AB = [(1.0, 0.0), (0.25, 1.0), (0.25, 2.0), (-0.5, 2.0)]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_resize_modes_flips_alpha_beta(log, mode):
    for k, (P, Hs, Ws, Hd, Wd) in enumerate(SHAPES):
        src = planes(P, Hs, Ws, 100 + k)
        old = planes(P, Hd, Wd, 200 + k)
        for flip in (False, True):
            for alpha, beta in AB:
                run_resize(log, f"shape{k}", src, Hd, Wd, mode, flip, alpha, beta, old)
        run_resize(log, f"shape{k}-nan-dst", src, Hd, Wd, mode, True, 0.75, 0.0, nan_dst=True)
    src = planes(6, 29, 41, 5)
    for m in (0, 1):   # a same-size resize is an exact flip
        _, got = run_resize(log, "same-size-flip", src, 29, 41, m, True)
        assert torch.equal(got, src.flip(-1))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_resize_at_the_grid_cap(log, mode):
    """Work of cap*256 - 1, cap*256 and cap*256 + 1 elements, as long rows, as single pixels and as short planes."""
    seen = set()
    for n in (cap() - 1, cap(), cap() + 1):
        for (P, Hs, Ws, Hd, Wd) in ((1, 1, 7, 1, n), (n, 2, 3, 1, 1), (1, 5, 3, n, 1)):
            run_resize(log, f"cap{n - cap():+d}", planes(P, Hs, Ws, n + Hs), Hd, Wd, mode, bool(n % 2), 0.5, 0.0)
            sg = dc.stream_grid(P * Hd * Wd, sms())
            seen.add((sg.capped, sg.iters))
    assert (False, 1) in seen and (True, 2) in seen, seen


def test_zoom_factors_and_scipys_black_edge(log):
    saw_fill = False
    for (H, W) in ((64, 48), (37, 53), (97, 129), (48, 48), (5, 3)):
        src = planes(3, H, W, H * W, 4.0)
        for s in (0.25, 0.5, 0.75, 1.25, 1.5, 1.75, 2.0, 2.25, 3.0):
            Hd, Wd = max(1, int(round(H * s))), max(1, int(round(W * s)))
            saw_fill |= bool(dc.zoom_fill_mask(H, W, Hd, Wd).any())
            run_resize(log, f"zoom{s}", src, Hd, Wd, 2, False, 1.0, 0.0)
        for (sh, sw) in ((0.25, 3.0), (3.0, 0.5)):
            run_resize(log, f"zoom{sh}x{sw}", src, max(1, int(round(H * sh))), max(1, int(round(W * sw))), 2, True, 0.5,
                       1.0, planes(3, max(1, int(round(H * sh))), max(1, int(round(W * sw))), 7))
    assert saw_fill, "the parameter list is meant to include a pair that triggers scipy's constant-fill edge"


def test_resize_64bit_index(log):
    """An output of more than 2^31 elements (8.6 GB of fp32), checked on sampled planes that include the last one."""
    free, _ = torch.cuda.mem_get_info()
    if free < 20 * 2**30:
        pytest.skip(f"needs 20 GB free, {free / 2**30:.1f} GB free")
    Hd = Wd = 256
    P = 2**31 // (Hd * Wd) + 1
    src = planes(P, 16, 16, 9)
    g = dc.FlatGuarded((P, Hd, Wd), torch.float32, device=DEV)
    s = src.to(DEV)
    lib.call("seg_resize_nchw_f32", lib.ptr(s), P, 16, 16, lib.ptr(g.view), Hd, Wd, 1, 1, 1.0, 0.0)
    torch.cuda.synchronize()
    assert P * Hd * Wd > 2**31
    for part in (g.buf[:g.lead], g.buf[g.lead + g.n:]):
        assert bool(dc.is_sentinel(part).all()), "guard word overwritten"
    usage = 0.0
    for p in (0, 1, P // 2, P - 2, P - 1):
        got = g.view[p:p + 1].cpu()
        dc.check_written(f"64-bit plane {p}", got)
        usage = max(usage, dc.check_resize(f"64-bit plane {p}", got, dc.resize_bound(src[p:p + 1], Hd, Wd, 1, True)))
    log(f"resize mode=1 64-bit {P}x16x16->{Hd}x{Wd} elements={P * Hd * Wd} sampled planes usage={usage:.4f}")
    del g, s
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ window_add, div
def run_window(log, case, src, Hd, Wd, y0, x0, h, w, flip, alpha, seed):
    P, Hs, Ws = src.shape
    old = planes(P, Hd, Wd, seed)
    s = src.contiguous().to(DEV)
    runs = []
    for _ in range(2):
        g = dc.FlatGuarded((P, Hd, Wd), torch.float32, device=DEV)
        g.view.copy_(old)
        lib.call("seg_window_add_nchw_f32", lib.ptr(s), P, Hs, Ws, lib.ptr(g.view), Hd, Wd, y0, x0, h, w, int(flip), float(alpha))
        torch.cuda.synchronize()
        dc.check_guards(case, g.buf, g.guard_mask())
        runs.append(g.view.cpu())
    assert torch.equal(bits(runs[0]), bits(runs[1])), f"{case}: not bit-reproducible"
    u = dc.check_window_add(case, runs[0], old, src, y0, x0, h, w, flip, alpha)
    log(f"window_add {case} {P}x{Hs}x{Ws} into {Hd}x{Wd} at ({y0},{x0}) {h}x{w} flip={int(flip)} usage={u:.4f}")
    return u


def test_window_add_at_every_border(log):
    src = planes(6, 20, 33, 1)
    Hd, Wd = 50, 60
    wins = [(0, 0, 20, 33), (0, 60 - 33, 20, 33), (50 - 20, 0, 20, 33), (50 - 20, 60 - 33, 20, 33), (7, 11, 20, 33),
            (7, 11, 13, 20), (49, 59, 1, 1), (0, 0, 1, 33), (0, 0, 20, 1), (30, 27, 20, 33)]
    for k, (y0, x0, h, w) in enumerate(wins):
        for flip in (False, True):
            run_window(log, f"win{k}", src, Hd, Wd, y0, x0, h, w, flip, 0.5, k)
    run_window(log, "whole", planes(2, 50, 60, 2), 50, 60, 0, 0, 50, 60, True, 1.0, 99)
    for n in (cap() - 1, cap(), cap() + 1):
        run_window(log, f"cap{n - cap():+d}", planes(1, 1, n, 3), 3, n + 2, 1, 2, 1, n, True, -0.25, 5)


def run_div(log, case, x, count):
    runs = []
    for _ in range(2):
        g = dc.FlatGuarded(tuple(x.shape), torch.float32, device=DEV)
        g.view.copy_(x)
        c = count.to(DEV)
        P, H, W = x.shape
        lib.call("seg_div_by_count_nchw_f32", lib.ptr(g.view), P, H, W, lib.ptr(c))
        torch.cuda.synchronize()
        dc.check_guards(case, g.buf, g.guard_mask())
        runs.append(g.view.cpu())
    assert torch.equal(bits(runs[0]), bits(runs[1])), f"{case}: not bit-reproducible"
    dc.check_div(case, runs[0], x, count)
    log(f"div_by_count {case} {tuple(x.shape)} exact")


def window_count(H, W):
    cnt = torch.zeros(H, W)
    for (y0, y1, x0, x1) in di.sliding_windows(H, W)[1]:
        cnt[y0:y1, x0:x1] += 1
    return cnt


def test_div_by_count_with_sliding_window_counts(log):
    for (H, W) in ((37, 53), (64, 48), (300, 20), (100, 30), (513, 513), (97, 129)):
        cnt = window_count(H, W)
        x = planes(5, H, W, H) * cnt
        run_div(log, f"{H}x{W}", x, cnt)
    cnt = torch.randint(0, 5, (1, cap() + 1), generator=torch.Generator().manual_seed(3)).float()
    for n in (cap() - 1, cap(), cap() + 1):
        x = planes(1, 1, n, n)
        x[:, cnt[:, :n] == 0] = 0.0
        run_div(log, f"cap{n - cap():+d}", x, cnt[:, :n].contiguous())


# ------------------------------------------------------------------------------------------------ label map
def run_labels(log, case, scores):
    N, C, H, W = scores.shape
    s = scores.contiguous().to(DEV)
    runs = []
    for _ in range(2):
        g = dc.FlatGuarded((N, H, W), torch.int64, device=DEV)
        lib.call("seg_argmax_nchw_f32", lib.ptr(s), N, C, H, W, lib.ptr(g.view))
        torch.cuda.synchronize()
        dc.check_guards(case, g.buf, g.guard_mask())
        dc.check_written(case, g.view)
        runs.append(g.view.cpu())
    assert torch.equal(runs[0], runs[1]), f"{case}: not bit-reproducible"
    n = dc.check_labels(case, runs[0], scores)
    log(f"argmax {case} {tuple(scores.shape)} exact near_zero_ties={n}")
    return n, runs[0]


def test_label_map_non_finite_ties_and_the_near_zero_tie(log):
    from test_data_check_cpu import label_columns
    s = label_columns()
    n, lab = run_labels(log, "columns", s)
    # the documented choice for a tie the float64 softmax cannot resolve: the larger score wins (the reference keeps 0)
    assert n == 1 and lab[0, 0, 13].item() == 1 and dc.softmax_labels(s)[0, 0, 13].item() == 0
    g = torch.Generator().manual_seed(5)
    r = torch.randn(2, 7, 19, 23, generator=g)
    r[:, 3] = r[:, 1]
    r[0, 2, 4, 5], r[1, 6, 0, 0], r[1, 0, 18, 22] = math.nan, math.inf, math.nan
    run_labels(log, "random", r)
    for n in (cap() - 1, cap(), cap() + 1):
        q = torch.randint(-3, 3, (1, 3, 1, n), generator=g).float()   # many ties
        run_labels(log, f"cap{n - cap():+d}", q)
        assert dc.stream_grid(n, sms()).capped == (n > cap())


# ------------------------------------------------------------------------------------------------ TTA pipeline
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inference.npz")
SCALES = [0.75, 1.0, 1.5]


def tta_images():
    g = np.load(GOLD)
    out = [("golden-a", torch.from_numpy(g["a/image"])), ("golden-b", torch.from_numpy(g["b/image"]))]
    for (H, W) in ((300, 20), (100, 30), (37, 53), (64, 48), (97, 129)):
        out.append((f"{H}x{W}", torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(H)) * 2 - 1))
    return out


@pytest.mark.parametrize("flip", [False, True])
def test_tta_pipeline_against_the_oracle(log, flip):
    C = 5
    model = oi.toy_model(C, seed=3)
    host_model = lambda t: model(t.to(DEV)).cpu()  # noqa: E731  the same GPU convolutions on both sides
    for name, img in tta_images():
        _, _, H, W = img.shape
        x = img.to(DEV)
        with torch.no_grad():
            for s in SCALES:   # the model sees identical inputs on both sides: the zoom is bit-exact against scipy here
                Hs, Ws = int(round(H * s)), int(round(W * s))
                if (Hs, Ws) != (H, W):
                    dz = di.ops.resize_nchw(x, Hs, Ws, zoom=True).cpu()[0]
                    assert torch.equal(bits(dz), bits(dc.scipy_zoom(img[0], Hs, Ws))), f"{name}: zoom {s} is not bit-exact"
            got = di.multi_scale_predict(model, x, SCALES, C, flip=flip)
            ref, mag = dc.tta_reference("ms", host_model, img, C, flip, SCALES)
            u, acc = dc.check_tta(f"ms {name} flip={flip}", got, ref, mag, len(SCALES) * (2 if flip else 1))
            free = dc.check_tta_labels(f"ms {name}", di.predict_labels(got), ref, acc)
            log(f"tta ms {name} flip={int(flip)} usage={u:.4f} label_free_pixels={free}")
            got = di.sliding_predict(model, x, C, flip=flip)
            ref, mag = dc.tta_reference("slide", host_model, img, C, flip)
            u, acc = dc.check_tta(f"slide {name} flip={flip}", got, ref, mag, dc.sliding_terms(H, W, flip))
            free = dc.check_tta_labels(f"slide {name}", di.predict_labels(got), ref, acc)
            nan = int(torch.isnan(ref[0]).sum())
            log(f"tta slide {name} flip={int(flip)} usage={u:.4f} label_free_pixels={free} uncovered={nan}")
            if name == "300x20":
                assert nan == 3600
