"""Self-tests of the convolution conformance checker (tests/conv_check.py), CPU only.

Acceptance: the checker passes correct results computed differently — the float64 reference rounded to the output type,
and ATen's float32 CPU convolution (another summation order).  Sensitivity: it rejects each planted defect a broken kernel
would produce, and names its coordinates.  The planted defects stand in for broken kernels, which are never run."""
import math

import pytest
import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

import conv_check as cc

# (N, H, W, C, K, R, stride, pad, dil): small shapes of the GPU sweep
SHAPES = [
    (2, 9, 11, 64, 48, 3, 1, 1, 1),
    (1, 17, 17, 72, 24, 3, 2, 1, 1),
    (1, 16, 16, 16, 24, 5, 1, 2, 1),
    (2, 13, 13, 56, 136, 1, 2, 0, 1),
    (1, 33, 33, 16, 8, 3, 1, 18, 18),
]
IDS = ["x".join(map(str, s)) for s in SHAPES]


def outsz(H, R, stride, pad, dil):
    return (H + 2 * pad - dil * (R - 1) - 1) // stride + 1


def operands(shape, seed=0):
    N, H, W, C, K, R, stride, pad, dil = shape
    return cc.make_x(N, H, W, C, seed), cc.make_w(K, C, R, R, seed + 10)


def to_bf16(t):
    return t.to(torch.bfloat16).double()


def to_f32(t):
    return t.float().double()


# ------------------------------------------------------------------------------------------------ acceptance
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_accepts_fprop(shape):
    N, H, W, C, K, R, stride, pad, dil = shape
    x, w = operands(shape)
    g = torch.Generator().manual_seed(5)
    bias = torch.randn(K, generator=g, dtype=torch.float64).float().double()
    r = cc.fprop_ref(x, w, stride, pad, dil, bias=bias)
    aten = cc.nhwc(F.conv2d(cc.nchw(x).float(), w.float(), bias.float(), stride, pad, dil)).double()
    assert cc.check_elements("fp32 ref", to_f32(r.ref), r, False) <= 1
    assert cc.check_elements("fp32 aten", aten, r, False) <= 1
    assert cc.check_elements("bf16 ref", to_bf16(r.ref), r, True) <= 1
    assert cc.check_elements("bf16 aten", to_bf16(aten), r, True) <= 1
    # beta = 0.5: the wgmma epilogue's staged rounding (bf16 conv, then + beta old, rounded again) is inside the bound
    old = to_bf16(torch.randn(r.ref.shape, generator=g, dtype=torch.float64))
    rb = cc.fprop_ref(x, w, stride, pad, dil, bias=bias, beta=0.5, old=old)
    staged = to_bf16(to_bf16(aten).float() + 0.5 * old.float())
    assert cc.check_elements("bf16 staged", staged, rb, True, staged=True) <= 1
    assert cc.check_elements("fp32 beta", to_f32(aten.float() + 0.5 * old.float()), rb, False) <= 1


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_accepts_dgrad(shape):
    N, H, W, C, K, R, stride, pad, dil = shape
    x, w = operands(shape)
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, R, stride, pad, dil)
    dy = cc.make_x(N, P, Q, K, 7)
    old = cc.make_x(N, H, W, C, 8)
    for beta in (0.0, 0.5):
        r = cc.dgrad_ref(dy, w, (N, H, W, C), stride, pad, dil, beta=beta, old=old)
        aten = cc.nhwc(nn_grad.conv2d_input((N, C, H, W), w.float(), cc.nchw(dy).float(), stride, pad, dil)).double()
        aten = aten + beta * old
        assert cc.check_elements("bf16 ref", to_bf16(r.ref), r, True) <= 1
        assert cc.check_elements("bf16 aten", to_bf16(aten), r, True) <= 1


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_accepts_wgrad(shape):
    N, H, W, C, K, R, stride, pad, dil = shape
    x, w = operands(shape)
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, R, stride, pad, dil)
    dy = cc.make_x(N, P, Q, K, 7)
    old = torch.randn(R * R, K, C, generator=torch.Generator().manual_seed(9), dtype=torch.float64).float().double()
    r = cc.wgrad_ref(dy, x, R, R, stride, pad, dil, old=old)
    aten = cc.pack_w(nn_grad.conv2d_weight(cc.nchw(x).float(), (K, C, R, R), cc.nchw(dy).float(), stride, pad, dil)).double()
    assert cc.check_elements("fp32 ref", to_f32(r.ref), r, False) <= 1
    assert cc.check_elements("fp32 aten", to_f32(aten + old), r, False, splits=4) <= 1


def tc_stats(y, K):
    """The wgmma epilogue's statistics of stored values y [M, K]: fp32 sums over stat_rows-row groups, the groups of a
    128-row tile added in fp32, the tiles added in fp64."""
    sr = cc.stat_rows_for(K)
    yf = y.float()
    M = y.shape[0]
    s1 = torch.zeros(K, dtype=torch.float64)
    s2 = torch.zeros(K, dtype=torch.float64)
    for m0 in range(0, M, cc.BM):
        a = torch.zeros(K, dtype=torch.float32)
        b = torch.zeros(K, dtype=torch.float32)
        for g0 in range(m0, min(m0 + cc.BM, M), sr):
            ga = torch.zeros(K, dtype=torch.float32)
            gb = torch.zeros(K, dtype=torch.float32)
            for r in range(g0, min(g0 + sr, M)):
                ga = ga + yf[r]
                gb = gb + yf[r] * yf[r]
            a, b = a + ga, b + gb
        s1 += a.double()
        s2 += b.double()
    return torch.cat([s1, s2])


@pytest.mark.parametrize("K", [48, 136, 320])
def test_accepts_statistics(K):
    y = to_bf16(cc.make_x(1, 9, 33, K, 3)).reshape(-1, K)
    assert cc.check_stats("tc", tc_stats(y, K), y, cc.stat_chain_tc(K)) <= 1
    f32 = torch.cat([y.float().sum(0), (y.float() ** 2).sum(0)]).double()
    assert cc.check_stats("f32 sum", f32, y, cc.stat_chain_simt(y.shape[0], K, 132)) <= 1


# ------------------------------------------------------------------------------------------------ sensitivity
def rejects(fn, *coords):
    with pytest.raises(AssertionError) as ei:
        fn()
    msg = str(ei.value)
    for c in coords:
        assert c in msg, f"{c!r} not in the failure message:\n{msg}"
    return msg


def old_max_norm_ok(got, ref, tol):
    """The max-normalised check the older tests use."""
    return ((got - ref).abs().max() / ref.abs().max()).item() <= tol


def test_rejects_two_ulp_move_in_low_magnitude_channel():
    shape = SHAPES[0]
    N, H, W, C, K, R, stride, pad, dil = shape
    x, w = operands(shape)
    r = cc.fprop_ref(x, w, stride, pad, dil)
    got = r.ref.to(torch.bfloat16)
    kq = r.mag.amax((0, 1, 2)).argmin().item()  # the lowest-magnitude output channel
    rel = torch.zeros_like(r.ref)
    rel[..., kq] = r.ref[..., kq].abs() / r.mag[..., kq]
    t = tuple(torch.nonzero(rel == rel.max())[0].tolist())
    bits = got.view(torch.int16)
    bits[t] += 2  # two bf16 ulps away from zero
    got = got.double()
    assert old_max_norm_ok(got, r.ref, 1e-2)
    rejects(lambda: cc.check_elements("2 ulp", got, r, True), f"n={t[0]}, h={t[1]}, w={t[2]}, c={t[3]}", "1 element(s)")


def test_rejects_dropped_largest_product_fprop_fp32():
    """fp32 fprop at the largest contraction of the sweep's fp32 fprop cases (3x3 x 304 channels = 2736)."""
    N, H, W, C, K, R, stride, pad, dil = 1, 7, 7, 304, 16, 3, 1, 1, 1
    x, w = cc.make_x(N, H, W, C, 1), cc.make_w(K, C, R, R, 2)
    r = cc.fprop_ref(x, w, stride, pad, dil)
    assert r.n == cc.LARGEST_FPROP_F32_N
    n_, h, w_, k = 0, 3, 3, 5
    cols = F.unfold(cc.nchw(x), R, dil, pad, stride)[0, :, h * W + w_]  # (c, r, s) order, as w[k].flatten()
    prods = cols * w[k].flatten()
    got = r.ref.float().double()
    got[n_, h, w_, k] -= prods[prods.abs().argmax()]
    rejects(lambda: cc.check_elements("dropped product", got, r, False), f"n=0, h={h}, w={w_}, c={k}")


def test_rejects_dropped_largest_product_wgrad_fp32():
    """fp32 wgrad at the largest pixel count of the sweep's wgrad cases."""
    n = cc.LARGEST_WGRAD_PIXELS
    H = W = math.isqrt(n)
    x, dy = cc.make_x(1, H, W, 8, 3), cc.make_x(1, H, W, 8, 4)
    r = cc.wgrad_ref(dy, x, 1, 1, 1, 0, 1)
    k, c = 3, 6
    prods = dy[0, :, :, k].flatten() * x[0, :, :, c].flatten()
    got = r.ref.float().double()
    got[0, k, c] -= prods[prods.abs().argmax()]
    rejects(lambda: cc.check_elements("dropped product", got, r, False, splits=132), f"tap=0, k={k}, c={c}")


def test_rejects_border_tap_reading_inside_the_image():
    shape = SHAPES[0]
    N, H, W, C, K, R, stride, pad, dil = shape
    x, w = operands(shape)
    r = cc.fprop_ref(x, w, stride, pad, dil)
    # output pixel (0, 0, 0): its tap (0, 0) reads the padding at (-1, -1); a broken kernel reads pixel (0, 0) instead
    delta = torch.einsum("c,kc->k", x[0, 0, 0], w[:, :, 0, 0])
    got = r.ref.clone()
    got[0, 0, 0] += delta
    rejects(lambda: cc.check_elements("border tap", to_bf16(got), r, True), "n=0, h=0, w=0")


def test_rejects_missing_k_chunk_in_one_tile():
    N, H, W, C, K, R, stride, pad, dil = 1, 19, 17, 200, 24, 3, 1, 1, 1
    x, w = cc.make_x(N, H, W, C, 1), cc.make_w(K, C, R, R, 2)
    r = cc.fprop_ref(x, w, stride, pad, dil)
    xm = torch.zeros_like(x)
    xm[..., 64:128] = x[..., 64:128]  # k-chunk 1 ...
    wm = torch.zeros_like(w)
    wm[:, :, 1, 1] = w[:, :, 1, 1]    # ... of the centre tap
    part = cc.fprop_ref(xm, wm, stride, pad, dil).staged.reshape(-1, K)
    got = r.ref.clone().reshape(-1, K)
    got[128:256] -= part[128:256]     # missing from the second row tile only
    got = got.reshape(r.ref.shape).float().double()
    msg = rejects(lambda: cc.check_elements("missing chunk", got, r, False), "n=0, h=7, w=9")  # row 128 = (7, 9)
    assert "n=0, h=0," not in msg  # the first tile is right


def test_rejects_zeroed_last_row_of_m_tail():
    N, H, W, C, K, R, stride, pad, dil = 1, 3, 43, 64, 64, 1, 1, 0, 1  # M = 129: one row in the tail tile
    x, w = cc.make_x(N, H, W, C, 1), cc.make_w(K, C, R, R, 2)
    r = cc.fprop_ref(x, w, stride, pad, dil)
    got = to_bf16(r.ref)
    got[0, 2, 42] = 0
    rejects(lambda: cc.check_elements("m tail", got, r, True), "n=0, h=2, w=42")


def test_rejects_overwritten_guard_word():
    for lead in (8, 13):
        g = cc.Guarded(2, 3, 5, 24, torch.bfloat16, lead=lead)
        g.view.copy_(torch.ones(2, 3, 5, 24))
        cc.check_guards("clean", g.buf, g.guard_mask())
        cc.check_written("clean", g.view)
        g.buf[1, 2, 4, lead + 24] = 0.0  # the first channel past the slice
        rejects(lambda: cc.check_guards("right guard", g.buf, g.guard_mask()), f"(1, 2, 4, {lead + 24})")
        g = cc.Guarded(2, 3, 5, 24, torch.float32, lead=lead)
        g.view.fill_(1.0)
        g.buf[2, 0, 0, lead] = 1.0  # the trailing guard image
        rejects(lambda: cc.check_guards("trailing image", g.buf, g.guard_mask()), f"(2, 0, 0, {lead})")
    f = cc.FlatGuarded((9, 8, 16), torch.float32, lead=1)
    f.view.fill_(0.0)
    f.buf[0] = 0.0
    rejects(lambda: cc.check_guards("flat", f.buf, f.guard_mask()), "(0,)")


def test_rejects_row_missing_from_one_channel_sum():
    K = 64
    y = to_bf16(cc.make_x(2, 33, 33, K, 3)).reshape(-1, K)
    s = tc_stats(y, K)
    c = 17
    row = y[:, c].abs().argmax()
    bad = s.clone()
    bad[c] -= y[row, c]
    exact = torch.cat([y.sum(0), (y * y).sum(0)])
    assert old_max_norm_ok(bad, exact, 2e-3)
    rejects(lambda: cc.check_stats("missing row", bad, y, cc.stat_chain_tc(K)), f"(sum, c={c})")


def test_rejects_unreachable_parity_class():
    """1x1 stride-2 dgrad: only the (even, even) input pixels receive taps; the three other parity classes are zeros
    (beta = 0) or beta * old."""
    N, H, W, C, K = 1, 9, 10, 16, 24
    w = cc.make_w(K, C, 1, 1, 2)
    dy = cc.make_x(N, 5, 5, K, 3)
    r = cc.dgrad_ref(dy, w, (N, H, W, C), 2, 0, 1)
    g = cc.Guarded(N, H, W, C, torch.bfloat16)
    g.view[:, ::2, ::2] = r.ref[:, ::2, ::2].to(torch.bfloat16)  # the other classes left at the sentinel
    rejects(lambda: cc.check_written("class left unwritten", g.view), "(0, 0, 1, 0)")
    old = cc.make_x(N, H, W, C, 4)
    rb = cc.dgrad_ref(dy, w, (N, H, W, C), 2, 0, 1, beta=0.5, old=old)
    got = to_bf16(rb.ref)
    got[:, 1::2] = old[:, 1::2]  # dx_old kept where 0.5 * dx_old was due
    rejects(lambda: cc.check_elements("class kept dx_old", got, rb, True), "n=0, h=1, w=0")
