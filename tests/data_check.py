"""Conformance checker for the kernels of seg_data.cu: the three augmentation kernels of the input pipeline (pad / crop /
flip / ToTensor / Normalize, with the random-scale resize, and with the rotation) and the four inference kernels of
test-time augmentation (resize_nchw, window_add, div_by_count, argmax), plus the TTA pipeline built from them.

Pure torch / numpy on the CPU, like conv_check.py, elementwise_check.py and dwconv_check.py, whose guarded buffers,
sentinels and Bound / check / check_exact it reuses: its own tests run without a GPU (test_data_check_cpu.py) and the GPU
sweep (test_data_conformance_gpu.py) feeds it what the kernels wrote.

Augmentation: bit-exact.  The reference is oracle/data.py's restatement of the reference pipeline (cv_resize_linear_f32,
cv_resize_nearest, cv_rotation_matrix, cv_warp_affine, then sample_tail's pad / crop / flip / np.uint8 / ToTensor /
Normalize), generalised here to a crop_h x crop_w crop.  Every step is either integer indexing, OpenCV's own fp32 or
fixed-point arithmetic, the np.uint8 truncation, or torchvision's fp32 division order, so no rounding is left to allow.
fused_emulation is the numpy transcription of augment_full_u8_kernel (per output pixel, no intermediate image), pinned to
the staged oracle by test_data_tail_oracle_cpu.py.

Per-element bounds of the fp32 inference kernels (u32 = 2^-24), "bound usage" as in conv_check: |got - ref| / e:

  resize_nchw, modes 0 / 1 (ATen bilinear, align_corners False / True).  Reference: the float64 blend with ATen's fp32
    source indices and lambdas (elementwise_check.lerp_axis, the kernel's own weights), times alpha, + beta dst.
    T = the same blend of |src| (the magnitude twin).  Roundings:
      inner lerps  w0 a + w1 b: two products and one sum, 2 u32 of |w0 a| + |w1 b| each;
      outer lerp   h0 i0 + h1 i1: the inner errors scaled by h (2 u32 T), two products and one sum (2 u32 T)  -> 4 u32 T;
      alpha * r: 1 more                                                                                        -> 5;
      beta * dst + v: the product and the sum, 2 u32 of |alpha| T + |beta dst|.
    K_RESIZE = 7 on |alpha| T + |beta dst| covers both parts; FMA contraction only removes roundings.  With beta = 0 the
    kernel stores v alone, so the reference ignores dst (a NaN-filled dst must be overwritten).
  resize_nchw, mode 2 (scipy.ndimage.zoom(order=1, prefilter=False)).  Reference: scipy itself, run at test time; the
    kernel and scipy both blend in float64 and round once to fp32, in different orders: 1 fp32 ulp of the zoomed value z
    is allowed, + K_ALPHA_BETA = 3 roundings (alpha z, beta dst, the sum) of |alpha z| + |beta dst|.  The constant-fill
    positions (coordinate > in - 1, mode='constant') are exact: such an element must equal fp32(beta dst), and scipy's z
    must be 0 there.
  window_add: dst + alpha src inside the window, one product and one sum: K_WINDOW = 2 on |dst| + |alpha src|; every
    element outside the window must keep its bits.
  div_by_count: one IEEE division: bit-exact (NaN where both sides are NaN: uncovered pixels are 0 / 0).
  argmax (label map): exact.  The reference is inference.py:156, softmax over the classes in float64, then argmax; the
    kernel's rule (label_rule): 0 where a pixel holds a NaN or +inf (the softmax column is all NaN and argmax returns the
    first NaN), else the first maximum score.  The two differ only where two top finite scores are closer than a float64
    softmax resolves (about 2^-53 relative to the top probability, so both scores under about 2e-9; the check allows 4e-9
    for the normalising division): the softmax rounds them to equal probabilities and keeps the first, the kernel takes
    the larger.  check_labels asserts that every disagreement is of that kind and counts them.

TTA pipeline (multi_scale_predict / sliding_predict against oracle/inference.py with the same deterministic stand-in
model): the oracle is the reference's own arithmetic (fp32 nn.Upsample on the CPU, float64 accumulation).  Magnitude
twin: the same oracle pipeline around |model|; every operation after the model is a non-negative-weight linear map, so
the twin bounds every intermediate.  Roundings per element, relative to T, for n accumulated terms (scales x flips, or
windows x flips): the device's resize of each term (5, as above, alpha included), its n sums into the fp32 total, and
the division by the count (1); the oracle's fp32 upsample (4) and its fp32 0.5 (a + b) (1).  K_TTA(n) = 11 + n, + 1
spare for the float64 accumulations of the oracle, which round too: 12 + n.  Labels must equal the reference's labels
wherever the reference's top-two margin exceeds the sum of the two scores' bounds (and wherever the scores are NaN).

Grid mirrors (aug_grid, stream_grid) copy seg_data.cu's host code, so the GPU sweep can assert which loops it reaches.
"""
import math
from collections import namedtuple

import numpy as np
import torch

from conv_check import GUARD, U32, FlatGuarded, check_guards, check_written, is_sentinel, sentinel_fill  # noqa: F401
from elementwise_check import Bound, bound, check, check_exact, lerp_axis, lerp_matrix  # noqa: F401
from oracle import data as od

THREADS = 256
BLOCKS_PER_SM = 8    # grid_for's cap and the augmentation kernels' share of blocks
AUG_U = 4            # pixels per thread and iteration of augment_u8_kernel
K_RESIZE = 7
K_ALPHA_BETA = 3
K_WINDOW = 2
NAMES_AUG = ("b", "c", "y", "x")
NAMES_LAB = ("b", "y", "x")
NAMES_PLANE = ("p", "y", "x")
NAMES_NCHW = ("n", "c", "y", "x")


def k_tta(n_terms):
    return 12 + n_terms


# ------------------------------------------------------------------------------------------------ grid mirrors
AugGrid = namedtuple("AugGrid", "per_image stride outer max_u iters")


def aug_grid(B, crop_h, crop_w, sms):
    """The augmentation launch (mirror of seg_augment_*_batch_u8): per_image blocks of 256 threads per image (blockIdx.y),
    ceil(8 SMs / B) clamped to [1, the blocks one pass needs].  stride = per_image * 256 pixels; augment_u8_kernel walks
    `outer` iterations of U = 4 pixels per thread (i0 + u stride) and reaches u = max_u; the scale and rotate kernels walk
    `iters` iterations of one pixel."""
    plane = crop_h * crop_w
    per_image = -(-(sms * BLOCKS_PER_SM) // B)
    per_image = max(1, min(per_image, -(-plane // THREADS)))
    stride = per_image * THREADS
    return AugGrid(per_image, stride, -(-plane // (stride * AUG_U)), min(AUG_U - 1, (plane - 1) // stride),
                   -(-plane // stride))


StreamGrid = namedtuple("StreamGrid", "blocks iters capped")


def stream_grid(work, sms):
    """grid_for(work, 256, 8): ceil(work / 256) blocks capped at 8 SMs, grid-stride over `work` elements."""
    cap = sms * BLOCKS_PER_SM
    need = max(1, -(-work // THREADS))
    blocks = min(need, cap)
    return StreamGrid(blocks, -(-work // (blocks * THREADS)), need > cap)


def grid_cap_elements(sms):
    """Elements one pass of a capped stream grid covers: cap * 256."""
    return sms * BLOCKS_PER_SM * THREADS


# ------------------------------------------------------------------------------------------------ augmentation
def tail_u8(image, label, crop_h, crop_w, y0, x0, flip):
    """sample_tail's pad / crop / flip for a crop_h x crop_w crop: (uint8 [crop_h, crop_w, 3], int64 [crop_h, crop_w] or
    None).  The padding is cv2.copyMakeBorder's constant 0, for the label too."""
    h, w = image.shape[:2]
    ph, pw = max(crop_h - h, 0), max(crop_w - w, 0)
    img = np.pad(image, ((0, ph), (0, pw), (0, 0)), mode="constant", constant_values=0)[y0:y0 + crop_h, x0:x0 + crop_w]
    lab = None
    if label is not None:
        lab = np.pad(np.asarray(label), ((0, ph), (0, pw)), mode="constant", constant_values=0)[y0:y0 + crop_h, x0:x0 + crop_w]
    if flip:
        img = np.fliplr(img)
        lab = None if lab is None else np.fliplr(lab)
    assert img.shape == (crop_h, crop_w, 3), (img.shape, crop_h, crop_w, y0, x0)
    return np.ascontiguousarray(img), (None if lab is None else np.array(lab, dtype=np.int64))


def normalise(u8, mean, std):
    """ToTensor + Normalize of uint8 [B, h, w, 3] as sample_tail computes them (fp32 / 255, - mean, / std)."""
    t = torch.from_numpy(np.ascontiguousarray(u8)).permute(0, 3, 1, 2).contiguous().to(torch.float32).div(255)
    m = torch.as_tensor(mean, dtype=torch.float32).view(1, -1, 1, 1)
    s = torch.as_tensor(std, dtype=torch.float32).view(1, -1, 1, 1)
    return t.sub_(m).div_(s)


def resized_sample(image, label, h, w, angle=None):
    """base_dataset.py:66-83 as oracle/data.py restates it: resize to h x w (float image, nearest label), then rotate by
    `angle` degrees about the centre; the float image is truncated to uint8 (np.uint8)."""
    img = od.cv_resize_linear_f32(image, w, h)
    lab = None if label is None else od.cv_resize_nearest(np.asarray(label), w, h)
    if angle is not None:
        M = od.cv_rotation_matrix((w / 2, h / 2), angle, 1.0)
        img = od.cv_warp_affine(img, M, w, h, linear=True)
        lab = None if lab is None else od.cv_warp_affine(lab, M, w, h, linear=False)
    return np.uint8(img), lab


def aug_sample_u8(kind, sample, crop_h, crop_w):
    """One sample of a batch in DeviceBatcher's format -> (uint8 crop, int64 label crop or None).
    kind "plain": (image, label, y0, x0, flip); "scale": (image, label, h, w, y0, x0, flip);
    "full": (image, label, h, w, angle, y0, x0, flip)."""
    if kind == "plain":
        img, lbl, y0, x0, flip = sample
    elif kind == "scale":
        im, lb, h, w, y0, x0, flip = sample
        img, lbl = resized_sample(im, lb, h, w)
    else:
        im, lb, h, w, angle, y0, x0, flip = sample
        img, lbl = resized_sample(im, lb, h, w, angle)
    return tail_u8(img, lbl, crop_h, crop_w, y0, x0, bool(flip))


def aug_reference(kind, samples, crop_h, crop_w, mean, std, want_labels=True):
    """(images fp32 [B, 3, crop_h, crop_w], labels int64 [B, crop_h, crop_w] or None).  A sample without a label in a
    labelled batch gets label 0 (the kernel's lbl_off < 0)."""
    u8, labs = [], []
    for s in samples:
        x, y = aug_sample_u8(kind, s, crop_h, crop_w)
        u8.append(x)
        labs.append(np.zeros((crop_h, crop_w), np.int64) if y is None else y)
    x = normalise(np.stack(u8), mean, std)
    return x, (torch.from_numpy(np.stack(labs)) if want_labels else None)


def check_augment(case, x, labels, x_ref, labels_ref):
    """Bit-exact images (no NaN can occur: std != 0 is checked by the host) and labels."""
    check_exact(case, "images", x, x_ref, NAMES_AUG)
    if labels_ref is not None:
        check_exact(case, "labels", labels, labels_ref, NAMES_LAB)
    else:
        assert labels is None, case


def fused_emulation(image, label, h, w, angle, crop, y0, x0, flip, mean, std, fault=None):
    """numpy transcription of augment_full_u8_kernel (seg_data.cu): per OUTPUT pixel, fixed-point rotated coordinates ->
    four taps of the resized image, each interpolated on the fly from the raw image -> truncate -> normalise.  No resized or
    rotated intermediate, exactly the kernel's operation order.  With angle None the rotation is the identity and this is
    augment_scale_u8_kernel.  crop: an int (square) or (crop_h, crop_w).  fault: a named seeded defect, for the checker's
    own tests ("round_label", "label_delta_16", "round_u8")."""
    from seg_b200.data import inverse_rotation
    crop_h, crop_w = (crop, crop) if isinstance(crop, int) else crop
    H, W = image.shape[:2]
    sx_scale, sy_scale = 1.0 / (w / W), 1.0 / (h / H)
    a11, a12, b1, a21, a22, b2 = inverse_rotation(w, h, angle)
    raw = image.astype(np.float32)
    f32 = np.float32

    def coord(d, scale, src, clamp):
        fv = ((d.astype(np.float64) + 0.5) * scale - 0.5).astype(np.float32)
        fl = np.floor(fv)
        s = fl.astype(np.int64)
        f = (fv - fl).astype(np.float32)
        if clamp:
            lo, hi = s < 0, s >= src - 1
            f = np.where(lo | hi, f32(0), f)
            s = np.where(lo, 0, np.where(hi, src - 1, s))
        return s, f

    def resized(ry, rx):  # float value of the resized image at integer (ry, rx); 0 outside
        ok = (ry >= 0) & (ry < h) & (rx >= 0) & (rx < w)
        ryc, rxc = np.clip(ry, 0, h - 1), np.clip(rx, 0, w - 1)
        sx, fx = coord(rxc, sx_scale, W, True)
        sy, fy = coord(ryc, sy_scale, H, False)
        sx1 = np.minimum(sx + 1, W - 1)
        y0c, y1c = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)
        ax0, ay0 = (f32(1) - fx)[..., None], (f32(1) - fy)[..., None]
        fx_, fy_ = fx[..., None], fy[..., None]
        h0 = raw[y0c, sx] * ax0 + raw[y0c, sx1] * fx_
        h1 = raw[y1c, sx] * ax0 + raw[y1c, sx1] * fx_
        return np.where(ok[..., None], h0 * ay0 + h1 * fy_, f32(0)).astype(np.float32)

    ys, xs = np.meshgrid(np.arange(crop_h), np.arange(crop_w), indexing="ij")
    xs = crop_w - 1 - xs if flip else xs
    dy, dx = ys + y0, xs + x0
    inside = (dy < h) & (dx < w)
    rnd = lambda v: np.rint(v).astype(np.int64)  # noqa: E731
    colX, colY = rnd(a11 * dx.astype(np.float64) * 1024.0), rnd(a21 * dx.astype(np.float64) * 1024.0)
    rowX, rowY = rnd((a12 * dy.astype(np.float64) + b1) * 1024.0), rnd((a22 * dy.astype(np.float64) + b2) * 1024.0)
    X, Y = rowX + 16 + colX, rowY + 16 + colY
    Xf, Yf = X >> 5, Y >> 5
    xi, yi = Xf >> 5, Yf >> 5
    fx, fy = (Xf & 31).astype(np.float32) / f32(32), (Yf & 31).astype(np.float32) / f32(32)
    w00, w01 = ((f32(1) - fy) * (f32(1) - fx))[..., None], ((f32(1) - fy) * fx)[..., None]
    w10, w11 = (fy * (f32(1) - fx))[..., None], (fy * fx)[..., None]
    v = resized(yi, xi) * w00 + resized(yi, xi + 1) * w01 + resized(yi + 1, xi) * w10 + resized(yi + 1, xi + 1) * w11
    if fault == "round_u8":
        v = np.rint(v)
    u8 = np.where(inside[..., None], np.clip(np.where(v > 0, v, 0).astype(np.int64), 0, 255), 0).astype(np.uint8)
    delta = 16 if fault == "label_delta_16" else 512
    Xn, Yn = (rowX + delta + colX) >> 10, (rowY + delta + colY) >> 10
    okl = inside & (Yn >= 0) & (Yn < h) & (Xn >= 0) & (Xn < w)
    lfloor = np.rint if fault == "round_label" else np.floor
    lx = np.minimum(lfloor(np.clip(Xn, 0, w - 1).astype(np.float64) * sx_scale).astype(np.int64), W - 1)
    ly = np.minimum(lfloor(np.clip(Yn, 0, h - 1).astype(np.float64) * sy_scale).astype(np.int64), H - 1)
    lab = np.zeros((crop_h, crop_w), np.int64) if label is None else np.where(okl, np.asarray(label)[ly, lx], 0).astype(np.int64)
    return normalise(u8[None], mean, std)[0], torch.from_numpy(lab)


# ------------------------------------------------------------------------------------------------ resize_nchw
def zoom_fill_mask(Hs, Ws, Hd, Wd):
    """[Hd, Wd] bool, the kernel's (and scipy's mode='constant') fill rule: float64 coordinate o (in - 1) / (out - 1)
    (1 where out == 1) greater than in - 1, on either axis; in unflipped output coordinates."""
    zh = (Hs - 1) / (Hd - 1) if Hd > 1 else 1.0
    zw = (Ws - 1) / (Wd - 1) if Wd > 1 else 1.0
    cy = np.arange(Hd, dtype=np.float64) * zh
    cx = np.arange(Wd, dtype=np.float64) * zw
    return torch.from_numpy((cy[:, None] > Hs - 1) | (cx[None, :] > Ws - 1))


def scipy_zoom(src, Hd, Wd):
    """scipy.ndimage.zoom(order=1, prefilter=False) of fp32 planes [P, Hs, Ws] to [P, Hd, Wd] (fp32, as scipy returns it
    for an fp32 input), asking for the zoom factor out / in, which scipy rounds back to the output size."""
    from scipy import ndimage
    P, Hs, Ws = src.shape
    z = ndimage.zoom(src.numpy(), (1.0, Hd / Hs, Wd / Ws), order=1, prefilter=False)
    assert z.shape == (P, Hd, Wd), (z.shape, (P, Hd, Wd))
    return torch.from_numpy(z)


def resize_bound(src, Hd, Wd, mode, flip=False, alpha=1.0, beta=0.0, old=None, zoomed=None):
    """Bound of dst = beta old + alpha [flip] resize(src) for src fp32 [P, Hs, Ws].  mode 0 / 1: ATen bilinear; mode 2:
    scipy's zoom (zoomed: a precomputed scipy_zoom of src, else it is computed here).  Fill elements of mode 2 carry a
    zero allowance around fp32(beta old): they must be exact."""
    P, Hs, Ws = src.shape
    a = float(np.float32(alpha))
    b = float(np.float32(beta))
    if mode in (0, 1):
        Ay, Ax = lerp_matrix(Hs, Hd, mode == 1), lerp_matrix(Ws, Wd, mode == 1)
        R = torch.einsum("oh,phw,qw->poq", Ay, src.double(), Ax)
        T = torch.einsum("oh,phw,qw->poq", Ay.abs(), src.double().abs(), Ax.abs())
        fill = None
    else:
        z = scipy_zoom(src, Hd, Wd) if zoomed is None else zoomed
        fill = zoom_fill_mask(Hs, Ws, Hd, Wd)
        zf = z[:, fill]
        if zf.numel() and not bool((zf == 0).all()):
            raise AssertionError(f"scipy's zoom is not 0 at the kernel's fill positions ({Hs}x{Ws} -> {Hd}x{Wd})")
        zd = z.double()
        ulp = (torch.nextafter(z.abs(), torch.tensor(math.inf)) - z.abs()).double()
        R, T = zd, None
    if flip:
        R = R.flip(-1)
        T = None if T is None else T.flip(-1)
        ulp = ulp.flip(-1) if mode == 2 else None
        fill = None if fill is None else fill.flip(-1)
    ref = a * R
    if mode == 2:
        acc = abs(a) * ulp + K_ALPHA_BETA * U32 * (a * R).abs()
    else:
        acc = K_RESIZE * U32 * abs(a) * T
    if b != 0.0:
        od_ = old.double()
        ref = ref + b * od_
        acc = acc + (K_ALPHA_BETA if mode == 2 else K_RESIZE) * U32 * (b * od_).abs()
    if fill is not None and bool(fill.any()):
        fv = (torch.tensor(b, dtype=torch.float32) * old.float()).double() if b != 0.0 else torch.zeros_like(ref)
        ref = torch.where(fill, fv, ref)
        acc = torch.where(fill, torch.zeros_like(acc), acc)
    return bound(ref, acc, False, NAMES_PLANE)


def check_resize(case, got, b):
    return check(case, "resize_nchw", got.reshape(b.ref.shape), b)


# ------------------------------------------------------------------------------------------------ window_add, div
def window_add_ref(old, src, y0, x0, h, w, flip=False, alpha=1.0):
    """old fp32 [P, Hd, Wd], src fp32 [P, Hs, Ws]: (Bound over the window, window slices)."""
    a = float(np.float32(alpha))
    s = src.double()
    if flip:
        s = s.flip(-1)
    s = s[:, :h, :w]
    o = old[:, y0:y0 + h, x0:x0 + w].double()
    return bound(o + a * s, K_WINDOW * U32 * (o.abs() + (a * s).abs()), False, NAMES_PLANE)


def check_window_add(case, got, old, src, y0, x0, h, w, flip=False, alpha=1.0):
    """Inside the window: the bound of one product and one sum.  Outside: the bits of `old`, unchanged."""
    got = got.detach().cpu()
    inside = torch.zeros(got.shape, dtype=torch.bool)
    inside[:, y0:y0 + h, x0:x0 + w] = True
    changed = (got.view(torch.int32) != old.view(torch.int32)) & ~inside
    n = int(changed.sum())
    if n:
        lines = [f"  (p, y, x)={tuple(ix)}: got={got[tuple(ix)].item():.9g} before={old[tuple(ix)].item():.9g}"
                 for ix in changed.nonzero()[:8].tolist()]
        raise AssertionError(f"{case}: window_add: {n} element(s) outside the window changed\n" + "\n".join(lines))
    b = window_add_ref(old, src, y0, x0, h, w, flip, alpha)
    return check(case, f"window_add (window at y0={y0}, x0={x0})", got[:, y0:y0 + h, x0:x0 + w], b)


def check_div(case, got, x, count):
    """x fp32 [P, H, W] / count fp32 [H, W]: IEEE division, bit-exact; NaN exactly where the division is NaN."""
    got = got.detach().cpu().float()
    ref = x.float() / count.float()
    bad = ~((got == ref) | (torch.isnan(got) & torch.isnan(ref)))
    n = int(bad.sum())
    if n:
        lines = [f"  (p, y, x)={tuple(ix)}: got={got[tuple(ix)].item():.9g} ref={ref[tuple(ix)].item():.9g}"
                 for ix in bad.nonzero()[:8].tolist()]
        raise AssertionError(f"{case}: div_by_count: {n} element(s) differ\n" + "\n".join(lines))


# ------------------------------------------------------------------------------------------------ label map
def softmax_labels(scores):
    """inference.py:156 on scores [N, C, H, W]: float64 softmax over C, then argmax (first NaN / first maximum)."""
    return torch.softmax(scores.double(), 1).argmax(1)


def label_rule(scores):
    """The kernel's documented rule: 0 where a pixel's scores hold NaN or +inf, else the first maximum score."""
    s = scores.float()
    bad = (torch.isnan(s) | (s == math.inf)).any(1)
    C = s.shape[1]
    mx = s.max(1, keepdim=True).values
    first = torch.where(s == mx, torch.arange(C).view(1, C, 1, 1), torch.full_like(s, C, dtype=torch.int64)).min(1).values
    return torch.where(bad, torch.zeros_like(first), first)


def check_labels(case, got, scores):
    """got int64 [N, H, W] must equal label_rule exactly; label_rule must equal the softmax reference except in columns
    whose two labels have equal float64 softmax probabilities (the unresolvable near-zero ties).  Returns their number."""
    scores = scores.detach().cpu()
    exp = label_rule(scores)
    check_exact(case, "labels", got.cpu(), exp, NAMES_LAB)
    ref = softmax_labels(scores)
    diff = exp != ref
    if bool(diff.any()):
        p = torch.softmax(scores.double(), 1)
        pe, pr = p.gather(1, exp.unsqueeze(1)).squeeze(1), p.gather(1, ref.unsqueeze(1)).squeeze(1)
        se, sr = scores.float().gather(1, exp.unsqueeze(1)).squeeze(1), scores.float().gather(1, ref.unsqueeze(1)).squeeze(1)
        other = diff & ~((pe == pr) & (se > sr) & (se.abs() < 4e-9) & (sr.abs() < 4e-9))
        if bool(other.any()):
            ix = other.nonzero()[0].tolist()
            raise AssertionError(f"{case}: label rule differs from the softmax reference at (n, y, x)={tuple(ix)}")
    return int(diff.sum())


# ------------------------------------------------------------------------------------------------ TTA pipeline
def abs_model(model):
    return lambda x: model(x).abs()


def tta_reference(kind, model, image, num_classes, flip, scales=None, device="cpu"):
    """(ref, mag) float64 [C, H, W] of oracle/inference.py's multi_scale_predict ("ms") or sliding_predict ("slide"),
    around `model` and around |model| (the magnitude twin)."""
    from oracle import inference as oi
    out = []
    for m in (model, abs_model(model)):
        with torch.no_grad():
            if kind == "ms":
                r = oi.multi_scale_predict(m, image, scales, num_classes, torch.device(device), flip=flip)
            else:
                r = oi.sliding_predict(m, image, num_classes, flip=flip)
        out.append(torch.from_numpy(np.asarray(r, dtype=np.float64)))
    return out[0], out[1]


def sliding_terms(H, W, flip):
    """Largest number of terms the sliding window accumulates into one pixel (windows covering it x flips)."""
    from seg_b200.inference import sliding_windows
    cover = np.zeros((H, W), np.int64)
    for (y0, y1, x0, x1) in sliding_windows(H, W)[1]:
        cover[y0:y1, x0:x1] += 1
    return int(cover.max()) * (2 if flip else 1)


def check_tta(case, got, ref, mag, n_terms):
    """Scores [C, H, W]: NaN exactly where the reference is NaN (pixels no window covers), elsewhere within
    K_TTA(n) u32 of the magnitude twin.  Returns (usage, per-element allowance)."""
    got = got.detach().to("cpu", torch.float64)
    nan_ref = torch.isnan(ref)
    wrong_nan = nan_ref != torch.isnan(got)
    if bool(wrong_nan.any()):
        ix = wrong_nan.nonzero()[0].tolist()
        raise AssertionError(f"{case}: scores: {int(wrong_nan.sum())} element(s) NaN on one side only, first (c, y, x)="
                             f"{tuple(ix)}: got={got[tuple(ix)].item():.9g} ref={ref[tuple(ix)].item():.9g}")
    acc = k_tta(n_terms) * U32 * mag
    keep = ~nan_ref
    b = bound(torch.where(keep, ref, torch.zeros_like(ref)), torch.where(keep, acc, torch.ones_like(acc)), False,
              ("c", "y", "x"))
    usage = check(case, "scores", torch.where(keep, got, torch.zeros_like(got)), b)
    return usage, acc


def check_tta_labels(case, got_labels, ref, acc):
    """The margin rule: got must equal softmax(ref).argmax wherever the reference's top-two margin exceeds the two scores'
    allowances, and at NaN pixels (label 0).  Returns the number of pixels the rule leaves free."""
    ref_lab = torch.softmax(ref.unsqueeze(0), 1).argmax(1)[0]
    got_labels = got_labels.detach().cpu()
    C = ref.shape[0]
    if C > 1:
        top = ref.topk(2, dim=0)
        a2 = acc.gather(0, top.indices)
        margin = top.values[0] - top.values[1]
        must = torch.isnan(margin) | (margin > a2[0] + a2[1])
    else:
        must = torch.ones(ref.shape[1:], dtype=torch.bool)
    bad = must & (got_labels != ref_lab)
    n = int(bad.sum())
    if n:
        lines = [f"  (y, x)={tuple(ix)}: got={got_labels[tuple(ix)].item()} ref={ref_lab[tuple(ix)].item()}"
                 for ix in bad.nonzero()[:8].tolist()]
        raise AssertionError(f"{case}: labels: {n} pixel(s) with a clear margin differ\n" + "\n".join(lines))
    return int((~must).sum())
