"""seg_augment_val_batch_u8 (the validation tail) and seg_augment_full_blur_batch_u8 (the training tail with the Gaussian
blur) against the staged CPU restatement of tests/val_blur_oracle.py — bit-exact — and against the reference's goldens;
DevicePrefetcher on a raw validation loader; refusals before any launch."""
import ctypes
import os

import numpy as np
import pytest
import torch

import val_blur_oracle as vo

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import lib
    from seg_b200.data import _FULL_ENTRY, DeviceBatcher, DevicePrefetcher, gaussian_taps, inverse_rotation

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data_val_blur.npz")
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
DEV = "cuda:0"


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def raw_label(rs, H, W, kind):
    if kind == "u8":
        return rs.randint(0, 256, (H, W)).astype(np.uint8)
    lb = rs.randint(0, 19, (H, W)).astype(np.int32)
    lb[rs.rand(H, W) < 0.2] = -1
    lb[rs.rand(H, W) < 0.2] = 255
    return lb


def check_val(b, samples, crop):
    x, y = b.stage_val(samples)
    torch.cuda.synchronize()
    assert x.shape == (len(samples), 3, crop, crop) and (y is None) == (samples[0][1] is None)
    for i, (im, lb) in enumerate(samples):
        rx, ry = vo.sample_val_tail(im, lb, crop, b.mean, b.std)
        assert torch.equal(bits(x[i].cpu()), bits(rx)), (i, im.shape, (x[i].cpu() - rx).abs().max().item())
        if lb is not None:
            assert torch.equal(y[i].cpu(), ry), (i, im.shape)
    return x, y


@pytest.mark.parametrize("kind", ["i32", "u8"])
def test_val_tail_cityscapes_frames(kind):
    """crop 480 on 1024 x 2048 frames (the shipped config's val_loader), B = 8, and portrait frames."""
    rs = np.random.RandomState(1 if kind == "i32" else 2)
    sizes = [(1024, 2048)] * 6 + [(2048, 1024), (1023, 2047)]
    samples = [(rs.randint(0, 256, (H, W, 3)).astype(np.uint8), raw_label(rs, H, W, kind)) for H, W in sizes]
    b = DeviceBatcher(MEAN, STD, 480, DEV, max_bytes=160 << 20)
    x, y = check_val(b, samples, 480)
    xi, yi = b.stage_val([(im, None) for im, _ in samples])  # images only
    assert yi is None and torch.equal(bits(xi), bits(x))


def test_val_tail_small_odd_frames_batch_16():
    rs = np.random.RandomState(3)
    b = DeviceBatcher([0.5, 0.25, 0.0], [0.5, 2.0, 0.125], 37, DEV, max_bytes=8 << 20)
    for rep in range(3):  # both staging slots get reused
        samples = []
        for k in range(16):
            H, W = [(int(rs.randint(1, 200)), int(rs.randint(1, 200))), (1, int(rs.randint(1, 90))), (int(rs.randint(1, 90)), 1),
                    (37, 37), (36, 38), (5, 9)][k % 6]
            samples.append((rs.randint(0, 256, (H, W, 3)).astype(np.uint8), raw_label(rs, H, W, ("i32", "u8")[(k + rep) % 2])))
        # a batch holds one label dtype per sample as the arena records it; mixing uint8 and int32 maps is allowed
        check_val(b, samples, 37)
    check_val(DeviceBatcher(MEAN, STD, 1, DEV), [(rs.randint(0, 256, (H, W, 3)).astype(np.uint8), raw_label(rs, H, W, "i32"))
                                                 for H, W in ((1, 1), (3, 7), (9, 2))], 1)


def test_val_tail_against_reference_goldens():
    g = np.load(GOLD)
    crop, mean, std = int(g["val_crop"]), g["mean"].tolist(), g["std"].tolist()
    n = int(g["n_val"])
    b = DeviceBatcher(mean, std, crop, DEV, max_bytes=1 << 20)
    x, y = b.stage_val([(g[f"v{i}/image"], g[f"v{i}/label"]) for i in range(n)])
    one_level = 1.0 / 255.0 / min(std) * 1.001
    for i in range(n):
        assert torch.equal(y[i].cpu(), torch.from_numpy(g[f"v{i}/y"])), i
        d = (x[i].cpu() - torch.from_numpy(g[f"v{i}/x"])).abs()
        assert d.max().item() <= one_level and (d > 0).float().mean().item() < 0.01, i


def test_prefetcher_on_a_raw_validation_loader():
    g = np.load(GOLD)
    crop, mean, std = int(g["val_crop"]), g["mean"].tolist(), g["std"].tolist()
    raw = [(g[f"v{i}/image"], g[f"v{i}/label"]) for i in range(int(g["n_val"]))]
    b = DeviceBatcher(mean, std, crop, DEV, max_bytes=1 << 20)
    want = [b.stage_val(raw[:3]), b.stage_val(raw[3:])]
    pf = DevicePrefetcher([raw[:3], raw[3:]], torch.device(DEV), batcher=b, val=True)
    assert len(pf) == 2
    got = list(pf)
    assert len(got) == 2
    for (x, y), (wx, wy) in zip(got, want):
        assert torch.equal(bits(x), bits(wx)) and torch.equal(y, wy)


# ------------------------------------------------------------------------------------------------ blur
def pack_full(samples):
    """Arena + seg_aug_full_entry table as DeviceBatcher packs them, for rectangular crops."""
    chunks, off = [], 0
    table = np.zeros(len(samples), dtype=_FULL_ENTRY)
    for k, (im, lb, h, w, angle, y0, x0, flip) in enumerate(samples):
        H, W = im.shape[:2]
        img_off = off
        chunks += [im.reshape(-1), np.zeros((-im.size) % 4, np.uint8)]
        off += im.size + (-im.size) % 4
        lbl_off, nb = off, lb.nbytes
        chunks += [lb.reshape(-1).view(np.uint8), np.zeros((-nb) % 4, np.uint8)]
        off += nb + (-nb) % 4
        table[k] = (img_off, lbl_off, 1.0 / (w / W), 1.0 / (h / H)) + inverse_rotation(w, h, angle) + \
            (H, W, h, w, y0, x0, int(flip), lb.dtype.itemsize)
    arena = torch.from_numpy(np.concatenate(chunks + [np.zeros(8, np.uint8)])).to(DEV)
    return arena, torch.from_numpy(table.view(np.uint8).copy()).to(DEV)


def c3(v):
    return (ctypes.c_float * 3)(*[float(x) for x in v])


def launch(name, arena, table, B, ch, cw, taps=None):
    x = torch.full((B, 3, ch, cw), float("nan"), device=DEV)
    y = torch.full((B, ch, cw), -7, dtype=torch.int64, device=DEV)
    args = (lib.ptr(arena), lib.ptr(table)) + ((lib.ptr(taps),) if taps is not None else ())
    lib.call(name, *args, B, ch, cw, c3(MEAN), c3(STD), lib.ptr(x), lib.ptr(y))
    torch.cuda.synchronize()
    return x.cpu(), y.cpu()


def blur_samples(rs, n, ch, cw, src=(20, 90)):
    out = []
    for k in range(n):
        H, W = int(rs.randint(*src)), int(rs.randint(*src))
        h, w = max(1, int(H * rs.uniform(0.5, 2.0))), max(1, int(W * rs.uniform(0.5, 2.0)))
        y0 = [0, max(h, ch) - ch, int(rs.randint(0, max(h, ch) - ch + 1))][k % 3]
        x0 = [max(w, cw) - cw, 0, int(rs.randint(0, max(w, cw) - cw + 1))][k % 3]
        out.append((rs.randint(0, 256, (H, W, 3)).astype(np.uint8), raw_label(rs, H, W, ("i32", "u8")[k % 2]), h, w,
                    [None, 0, -10, 7, 10][k % 5], y0, x0, bool((k // 2) % 2)))
    return out


def sigma_bands(rs, n):
    """sigma < 0.606 (k = 1), just above the k = 3 threshold, the middle and the top of random.random()'s range"""
    bands = [lambda: float(rs.uniform(0, 0.6)), lambda: 2 / 3.3 + 1e-9, lambda: float(rs.uniform(0.61, 1.0)), lambda: 0.9999999]
    return [bands[k % 4]() for k in range(n)]


def check_blur(samples, sigmas, ch, cw):
    B = len(samples)
    arena, table = pack_full(samples)
    taps = torch.tensor([gaussian_taps(s) for s in sigmas], dtype=torch.float32, device=DEV)
    x, y = launch("seg_augment_full_blur_batch_u8", arena, table, B, ch, cw, taps)
    x2, y2 = launch("seg_augment_full_blur_batch_u8", arena, table, B, ch, cw, taps)
    assert torch.equal(bits(x), bits(x2)) and torch.equal(y, y2), "not bit-reproducible"
    for i, (s, sg) in enumerate(zip(samples, sigmas)):
        im, lb, h, w, angle, y0, x0, flip = s
        rx, ry = vo.sample_blur_tail(im, lb, h, w, (ch, cw), y0, x0, flip, MEAN, STD, angle, sg)
        assert torch.equal(bits(x[i]), bits(rx)), (i, ch, cw, sg, (x[i] - rx).abs().max().item())
        assert torch.equal(y[i], ry), (i, ch, cw)
    return arena, table, x, y


@pytest.mark.parametrize("crop", [(40, 40), (380, 380), (17, 300), (300, 17), (33, 65)])
def test_blurred_tail_every_sigma_band_flip_on_and_off(crop):
    rs = np.random.RandomState(sum(crop))
    ch, cw = crop
    n = 12 if max(crop) < 300 else 8
    src = (20, 90) if max(crop) < 300 else (200, 500)
    samples = blur_samples(rs, n, ch, cw, src)
    sigmas = sigma_bands(rs, n)
    assert {vo.blur_ksize(s) for s in sigmas} == {1, 3} and {s[7] for s in samples} == {False, True}
    check_blur(samples, sigmas, ch, cw)


@pytest.mark.parametrize("crop", [(1, 1), (1, 3), (3, 1), (2, 2), (2, 5), (1, 40)])
def test_blurred_tail_tiny_crops_where_reflect101_folds(crop):
    rs = np.random.RandomState(7 + crop[0] * 10 + crop[1])
    ch, cw = crop
    samples = blur_samples(rs, 8, ch, cw, (1, 12))
    check_blur(samples, sigma_bands(rs, 8), ch, cw)


def test_k1_samples_equal_the_unblurred_kernel_bytes():
    rs = np.random.RandomState(9)
    for ch, cw in ((64, 80), (1, 3), (33, 33)):
        samples = blur_samples(rs, 10, ch, cw)
        arena, table = pack_full(samples)
        ident = torch.tensor([[1.0, 0.0]] * len(samples), dtype=torch.float32, device=DEV)
        xb, yb = launch("seg_augment_full_blur_batch_u8", arena, table, len(samples), ch, cw, ident)
        xf, yf = launch("seg_augment_full_batch_u8", arena, table, len(samples), ch, cw)
        assert torch.equal(bits(xb), bits(xf)) and torch.equal(yb, yf), (ch, cw)


def test_stage_full_with_sigmas_against_reference_goldens():
    g = np.load(GOLD)
    crop, mean, std = int(g["crop"]), g["mean"].tolist(), g["std"].tolist()
    n = int(g["n_train"])
    samples = [(g[f"t{i}/image"], g[f"t{i}/label"]) + tuple(int(v) for v in g[f"t{i}/draw"][:3]) +
               tuple(int(v) for v in g[f"t{i}/draw"][3:]) for i in range(n)]
    sigmas = [float(g[f"t{i}/sigma"]) for i in range(n)]
    b = DeviceBatcher(mean, std, crop, DEV, max_bytes=1 << 20)
    x, y = b.stage_full(samples, sigmas)
    one_level = 1.0 / 255.0 / min(std) * 1.001
    for i, s in enumerate(samples):
        rx, ry = vo.sample_blur_tail(s[0], s[1], s[2], s[3], crop, s[5], s[6], bool(s[7]), mean, std, s[4], sigmas[i])
        assert torch.equal(bits(x[i].cpu()), bits(rx)) and torch.equal(y[i].cpu(), ry), i
        assert torch.equal(y[i].cpu(), torch.from_numpy(g[f"t{i}/y"])), i
        d = (x[i].cpu() - torch.from_numpy(g[f"t{i}/x"])).abs()
        assert d.max().item() <= one_level and (d > 0).float().mean().item() < 0.01, i
    # no sample blurred (k = 1 everywhere, or no sigmas): the unblurred kernel's bytes
    x1, y1 = b.stage_full(samples, [0.1] * n)
    x0, y0 = b.stage_full(samples)
    assert torch.equal(bits(x1), bits(x0)) and torch.equal(y1, y0)


def test_refusals_raise_before_any_launch():
    im = np.zeros((4, 5, 3), np.uint8)
    lb = np.zeros((4, 5), np.int32)
    n0 = lib.launch_count()
    for crop in (None, 0):
        with pytest.raises(ValueError, match="crop_size"):
            DeviceBatcher(MEAN, STD, crop, DEV)
    b = DeviceBatcher(MEAN, STD, 8, DEV, max_bytes=1 << 20)
    bad = [[(im, lb, 0)], [(im, np.zeros((5, 4), np.int32))], [(im[..., :2], None)], [(im, lb), (im, None)],
           [(np.zeros((0, 5, 3), np.uint8), None)]]
    for s in bad:
        with pytest.raises(ValueError, match="stage_val"):
            b.stage_val(s)
    s = (im, lb, 20, 30, 5, 0, 0, False)
    with pytest.raises(ValueError, match="crop origin"):
        b.stage_full([(im, lb, 20, 30, 5, -2, 0, False)], [0.8])
    with pytest.raises(ValueError, match="crop origin"):
        b.stage_full([(im, lb, 20, 30, 5, 0, 23, False)], [0.8])
    with pytest.raises(ValueError, match="blur sigmas"):
        b.stage_full([s, s], [0.8])
    with pytest.raises(ValueError, match="3x3"):
        b.stage_full([s], [1.3])
    arena, table = pack_full([s])
    taps = torch.tensor([[1.0, 0.0]], device=DEV)
    out = torch.empty(3 * 64, device=DEV)
    with pytest.raises(RuntimeError, match="bad batch"):
        lib.call("seg_augment_full_blur_batch_u8", lib.ptr(arena), lib.ptr(table), lib.ptr(taps), 0, 8, 8, c3(MEAN), c3(STD),
                 lib.ptr(out), None)
    with pytest.raises(RuntimeError, match="null pointer"):
        lib.call("seg_augment_full_blur_batch_u8", lib.ptr(arena), lib.ptr(table), None, 1, 8, 8, c3(MEAN), c3(STD),
                 lib.ptr(out), None)
    with pytest.raises(RuntimeError, match="bad batch"):
        lib.call("seg_augment_val_batch_u8", lib.ptr(arena), lib.ptr(table), 65536, 8, 8, c3(MEAN), c3(STD), lib.ptr(out), None)
    torch.cuda.synchronize()
    assert lib.launch_count() == n0, "a refused call launched a kernel"
