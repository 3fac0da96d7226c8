"""Self-tests of the depthwise conformance checker (tests/dwconv_check.py), CPU only.

Acceptance: the checker passes correct results computed differently — the float64 reference rounded to the output type,
and ATen's float32 grouped convolution (another summation order).  Sensitivity: it rejects each planted defect a broken
kernel would produce, and names its coordinates.  The planted defects stand in for broken kernels, which are never run.
The statistics cases emulate the forward kernel's fp32 summation order on the grid dw_grid gives for 132 SMs (an H100
SXM): sums of the stored (bf16) outputs pass, sums of the unrounded fp32 outputs do not."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

import cpu_emulation as emu
import dwconv_check as dc

SMS = 132
# (N, H, W, C, stride, pad, dil): small shapes of the GPU sweep, each geometry edge once
SHAPES = [
    (2, 9, 11, 64, 1, 1, 1),
    (1, 17, 16, 72, 2, 1, 1),
    (2, 13, 13, 24, 1, 2, 2),
    (1, 16, 17, 16, 2, 4, 4),
    (1, 3, 5, 8, 1, 4, 4),     # map smaller than the dilation: only the centre tap is in range
    (1, 10, 9, 16, 2, 0, 1),   # pad 0, stride 2: the last row / column is reached by no tap
    (1, 9, 9, 16, 1, 3, 2),    # pad != dil
]
IDS = ["x".join(map(str, s)) for s in SHAPES]


def to_bf16(t):
    return t.to(torch.bfloat16).double()


def to_f32(t):
    return t.float().double()


def operands(shape, seed=0):
    N, H, W, C, stride, pad, dil = shape
    P, Q = dc.outsz(H, stride, pad, dil), dc.outsz(W, stride, pad, dil)
    return dc.make_x(N, H, W, C, seed), dc.make_w9(C, seed + 10), dc.make_x(N, P, Q, C, seed + 20)


def aten_fprop(x, w9, stride, pad, dil):
    C = x.shape[-1]
    return dc.nhwc(F.conv2d(dc.nchw(x).float(), dc.w9_to_oihw(w9).float(), None, stride, pad, dil, groups=C)).double()


def aten_dgrad(dy, w9, x_shape, stride, pad, dil):
    N, H, W, C = x_shape
    return dc.nhwc(nn_grad.conv2d_input((N, C, H, W), dc.w9_to_oihw(w9).float(), dc.nchw(dy).float(), stride, pad, dil,
                                        groups=C)).double()


def aten_wgrad(dy, x, stride, pad, dil):
    C = x.shape[-1]
    return dc.oihw_to_w9(nn_grad.conv2d_weight(dc.nchw(x).float(), (C, 1, 3, 3), dc.nchw(dy).float(), stride, pad, dil,
                                               groups=C)).double()


def kernel_stats(y, sms=SMS):
    """The forward kernel's statistics of per-row values y [M, C], in its order: thread (block b, lane l) adds rows
    b rows_par + l + k gx rows_par in fp32, the block adds its lanes in fp32, the blocks' partials are added in fp64."""
    M, C = y.shape
    gx, _, rp = dc.dw_grid(M, C, sms)
    L = -(-M // (gx * rp))
    yp = torch.cat([y.float(), torch.zeros(L * gx * rp - M, C)]).view(L, gx, rp, C)
    t1 = torch.zeros(gx, rp, C)
    t2 = torch.zeros(gx, rp, C)
    for k in range(L):
        t1 = t1 + yp[k]
        t2 = t2 + yp[k] * yp[k]
    b1 = torch.zeros(gx, C)
    b2 = torch.zeros(gx, C)
    for r in range(rp):
        b1 = b1 + t1[:, r]
        b2 = b2 + t2[:, r]
    return torch.cat([b1.double().sum(0), b2.double().sum(0)])


# ------------------------------------------------------------------------------------------------ acceptance
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_accepts_fprop(shape):
    N, H, W, C, stride, pad, dil = shape
    x, w9, _ = operands(shape)
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    assert dc.check_fprop("bf16 ref", to_bf16(b.ref), b) <= 1
    assert dc.check_fprop("bf16 aten", to_bf16(aten_fprop(x, w9, stride, pad, dil)), b) <= 1


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_accepts_dgrad(shape):
    N, H, W, C, stride, pad, dil = shape
    x, w9, dy = operands(shape)
    old = dc.make_x(N, H, W, C, 8)
    aten = aten_dgrad(dy, w9, x.shape, stride, pad, dil)
    for beta in (0.0, 0.5, 1.0):
        b = dc.dgrad_ref(dy, w9, x.shape, stride, pad, dil, beta=beta, old=old)
        assert dc.check_dgrad("bf16 ref", to_bf16(b.ref), b) <= 1
        assert dc.check_dgrad("bf16 aten", to_bf16(aten.float() + beta * old.float()), b) <= 1
    # the kernel's gather form (the formulation the defect tests below break) agrees with the reference
    assert dc.check_dgrad("gather", to_bf16(dgrad_gather(dy, w9, x.shape, stride, pad, dil)),
                          dc.dgrad_ref(dy, w9, x.shape, stride, pad, dil)) <= 1


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_accepts_wgrad(shape):
    N, H, W, C, stride, pad, dil = shape
    x, w9, dy = operands(shape)
    M = dy.shape[0] * dy.shape[1] * dy.shape[2]
    chain = dc.wgrad_chain(M, C, SMS)
    old = to_f32(torch.randn(9, C, generator=torch.Generator().manual_seed(9), dtype=torch.float64))
    aten = aten_wgrad(dy, x, stride, pad, dil)
    for beta in (0.0, 0.5, 1.0):
        b = dc.wgrad_ref(dy, x, stride, pad, dil, chain, beta=beta, old=old)
        assert dc.check_wgrad("fp32 ref", to_f32(b.ref), b) <= 1
        assert dc.check_wgrad("fp32 aten", to_f32(beta * old.float() + aten.float()), b) <= 1


def test_accepts_pack_and_unpack():
    C = 40
    w = torch.randn(C, 1, 3, 3, generator=torch.Generator().manual_seed(1)).double()
    dc.check_pack("pack", dc.oihw_to_w9(w).clone(), w)
    g9 = to_f32(torch.randn(9, C, generator=torch.Generator().manual_seed(2), dtype=torch.float64))
    old = to_f32(torch.randn(C, 1, 3, 3, generator=torch.Generator().manual_seed(3), dtype=torch.float64))
    for beta in (0.0, 0.5, 1.0):
        b = dc.unpack_ref(g9, beta, old)
        assert dc.check_unpack("unpack", to_f32(beta * old.float() + dc.w9_to_oihw(g9).float()), b) <= 1


@pytest.mark.parametrize("case", dc.XCEPTION_CASES[::5] + [(8, 1, 1), (2056, 2, 1)], ids=lambda c: "x".join(map(str, c)))
def test_accepts_statistics_of_the_stored_output(case):
    N, H, W, C, stride, pad, dil = dc.xception_shape(*case)
    x, w9, _ = operands((N, H, W, C, stride, pad, dil))
    y = to_bf16(aten_fprop(x, w9, stride, pad, dil)).reshape(-1, C)
    assert dc.check_stats("stored", kernel_stats(y), y, dc.stat_chain_dw(y.shape[0], C, SMS)) <= 1


def test_emulated_dwconv_statistics_are_of_the_stored_output():
    """cpu_emulation.dwconv_fwd, which the engine tests run in place of the kernel, sums y as stored."""
    N, H, W, C, stride, pad, dil = dc.xception_shape(728, 1, 2)
    x, w9, _ = operands((N, H, W, C, stride, pad, dil))
    st = torch.zeros(2 * C, dtype=torch.float64)
    y = emu.dwconv_fwd(x.to(torch.bfloat16), w9.float(), stride, pad, dil, stats=st)
    assert dc.check_stats("emulation", st, y.double().reshape(-1, C), dc.stat_chain_dw(N * H * W, C, SMS)) <= 1


# ------------------------------------------------------------------------------------------------ sensitivity
def rejects(fn, *coords):
    with pytest.raises(AssertionError) as ei:
        fn()
    msg = str(ei.value)
    for c in coords:
        assert c in msg, f"{c!r} not in the failure message:\n{msg}"
    return msg


def planted(check, good, bad, b, channels=None):
    """The whole defective output must be rejected; then the defect is planted at the one element where it is most
    visible (in the given channels), and that element alone must be rejected, by its coordinates."""
    rejects(lambda: check("global", bad, b))
    u = (bad - b.ref).abs() / (b.rnd + b.acc)
    if channels is not None:
        keep = torch.zeros_like(u, dtype=torch.bool)
        keep[..., channels] = True
        u = torch.where(keep, u, torch.zeros_like(u))
    t = tuple(torch.nonzero(u == u.max())[0].tolist())
    got = good.clone()
    got[t] = bad[t]
    coords = ", ".join(f"{n}={v}" for n, v in zip(b.names, t))
    rejects(lambda: check("one element", got, b), coords, "1 element(s)")


def low_channels(C, seed):
    """The channels of make_x's lowest per-channel magnitude (2^-9)."""
    return torch.nonzero(dc.channel_scales(C, seed + 1) == 2.0 ** -9).flatten().tolist()


def test_rejects_dropped_tap():
    shape = SHAPES[0]
    N, H, W, C, stride, pad, dil = shape
    x, w9, _ = operands(shape)
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    w_bad = w9.clone()
    w_bad[5] = 0  # tap (r, s) = (1, 2)
    bad = to_bf16(dc.fprop_ref(x, w_bad, stride, pad, dil).ref)
    planted(dc.check_fprop, to_bf16(b.ref), bad, b, low_channels(C, 0))


def test_rejects_transposed_taps():
    shape = SHAPES[2]
    N, H, W, C, stride, pad, dil = shape
    x, w9, _ = operands(shape)
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    w_t = w9.view(3, 3, C).transpose(0, 1).reshape(9, C)  # tap (r, s) takes (s, r)'s weight
    assert not torch.equal(w_t, w9)
    planted(dc.check_fprop, to_bf16(b.ref), to_bf16(dc.fprop_ref(x, w_t, stride, pad, dil).ref), b)


def test_rejects_dilation_on_one_axis_only():
    N, H, W, C, stride, pad, dil = 1, 13, 13, 24, 1, 2, 2
    x, w9, _ = operands((N, H, W, C, stride, pad, dil))
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    # rows dilated, columns not (the padding follows so that the output size is the same)
    bad = dc.nhwc(F.conv2d(dc.nchw(x), dc.w9_to_oihw(w9), None, stride, (pad, 1), (dil, 1), groups=C))
    assert bad.shape == b.ref.shape
    planted(dc.check_fprop, to_bf16(b.ref), to_bf16(bad), b)


def test_rejects_padding_off_by_one():
    shape = SHAPES[1]  # stride 2
    N, H, W, C, stride, pad, dil = shape
    x, w9, _ = operands(shape)
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    P, Q = b.ref.shape[1:3]
    bad = dc.nhwc(F.conv2d(dc.nchw(x), dc.w9_to_oihw(w9), None, stride, pad + 1, dil, groups=C))[:, :P, :Q]
    planted(dc.check_fprop, to_bf16(b.ref), to_bf16(bad), b)


def dgrad_gather(dy, w9, x_shape, stride, pad, dil, parity=True):
    """The data gradient in dwconv_bwd_data_kernel's gather form: input pixel (ih, iw) takes tap (r, s) from output
    pixel (th / stride, tw / stride), th = ih + pad - r dil, when th is a non-negative multiple of the stride (and the
    same for the columns).  parity=False drops the multiple-of-stride test (a parity-class defect)."""
    N, H, W, C = x_shape
    P, Q = dy.shape[1:3]
    dx = torch.zeros(x_shape, dtype=torch.float64)

    def src(i, k):
        t = i + pad - k * dil
        if t < 0 or (parity and t % stride):
            return None
        return t // stride

    for ih in range(H):
        for iw in range(W):
            for r in range(3):
                p = src(ih, r)
                if p is None or p >= P:
                    continue
                for s in range(3):
                    q = src(iw, s)
                    if q is None or q >= Q:
                        continue
                    dx[:, ih, iw] += dy[:, p, q] * w9[3 * r + s]
    return dx


def test_rejects_stride2_parity_error_in_dgrad():
    shape = SHAPES[1]
    N, H, W, C, stride, pad, dil = shape
    x, w9, dy = operands(shape)
    b = dc.dgrad_ref(dy, w9, x.shape, stride, pad, dil)
    bad = to_bf16(dgrad_gather(dy, w9, x.shape, stride, pad, dil, parity=False))
    planted(dc.check_dgrad, to_bf16(b.ref), bad, b, low_channels(C, 0))


def test_rejects_shifted_channel_group():
    shape = SHAPES[0]
    N, H, W, C, stride, pad, dil = shape
    x, w9, _ = operands(shape)
    b = dc.fprop_ref(x, w9, stride, pad, dil)
    xs = x.clone()
    xs[..., 8:16] = x[..., 16:24]  # group 1 reads group 2's activations
    planted(dc.check_fprop, to_bf16(b.ref), to_bf16(dc.fprop_ref(xs, w9, stride, pad, dil).ref), b)


def test_rejects_ignored_beta():
    shape = SHAPES[3]
    N, H, W, C, stride, pad, dil = shape
    x, w9, dy = operands(shape)
    old = dc.make_x(N, H, W, C, 8)
    for beta in (0.5, 1.0):
        b = dc.dgrad_ref(dy, w9, x.shape, stride, pad, dil, beta=beta, old=old)
        planted(dc.check_dgrad, to_bf16(b.ref), to_bf16(dc.dgrad_ref(dy, w9, x.shape, stride, pad, dil).ref), b)
        M = dy.shape[0] * dy.shape[1] * dy.shape[2]
        oldw = to_f32(torch.randn(9, C, generator=torch.Generator().manual_seed(9), dtype=torch.float64))
        bw = dc.wgrad_ref(dy, x, stride, pad, dil, dc.wgrad_chain(M, C, SMS), beta=beta, old=oldw)
        planted(dc.check_wgrad, to_f32(bw.ref), to_f32(bw.ref - beta * oldw), bw)
        g9 = to_f32(torch.randn(9, C, generator=torch.Generator().manual_seed(2), dtype=torch.float64))
        oldu = to_f32(torch.randn(C, 1, 3, 3, generator=torch.Generator().manual_seed(3), dtype=torch.float64))
        bu = dc.unpack_ref(g9, beta, oldu)
        planted(dc.check_unpack, to_f32(bu.ref), dc.w9_to_oihw(g9), bu)


def test_rejects_dropped_pixel_in_wgrad_at_the_longest_chain():
    """One pixel's largest product left out of one tap of one channel, with the bound widened to the longest chain and
    the most pixels of the GPU sweep's weight-gradient cases."""
    H = W = 547
    C = 8
    assert H * W <= dc.LARGEST_DW_WGRAD_PIXELS < (H + 1) * (W + 1)
    x, dy = dc.make_x(1, H, W, C, 3), dc.make_x(1, H, W, C, 4)
    b = dc.wgrad_ref(dy, x, 1, 1, 1, dc.LARGEST_DW_WGRAD_CHAIN)
    t, c = 4, 6  # the centre tap: every pixel contributes
    prods = dy[0, :, :, c].flatten() * x[0, :, :, c].flatten()
    got = to_f32(b.ref)
    got[t, c] -= prods[prods.abs().argmax()]
    rejects(lambda: dc.check_wgrad("dropped pixel", got, b), f"tap={t}, c={c}", "1 element(s)")


def test_rejects_unwritten_element_and_overwritten_guard():
    for lead in (8, 16):
        g = dc.Guarded(2, 3, 5, 24, torch.bfloat16, lead=lead)
        g.view.copy_(torch.ones(2, 3, 5, 24))
        dc.check_guards("clean", g.buf, g.guard_mask())
        dc.check_written("clean", g.view)
        dc.sentinel_fill(g.view[1, 2, 3, 17:18])
        rejects(lambda: dc.check_written("unwritten", g.view), "(1, 2, 3, 17)")
        g.buf[0, 1, 4, lead - 1] = 0.0  # the last guard channel before the slice
        rejects(lambda: dc.check_guards("left guard", g.buf, g.guard_mask()), f"(0, 1, 4, {lead - 1})")
    f = dc.FlatGuarded((9, 16), torch.float32)
    f.view.fill_(0.0)
    dc.check_guards("clean", f.buf, f.guard_mask())
    f.buf[-1] = 0.0
    rejects(lambda: dc.check_guards("flat", f.buf, f.guard_mask()), f"({f.buf.numel() - 1},)")


@pytest.mark.parametrize("case", dc.XCEPTION_CASES, ids=lambda c: "x".join(map(str, c)))
def test_rejects_statistics_of_the_unrounded_output(case):
    """The forward's statistics summed from the fp32 values before they are rounded to bf16, in the kernel's order, are
    not the statistics of the stored output that bn_apply normalises: rejected at every statistics shape of the
    sweep's Xception layers."""
    N, H, W, C, stride, pad, dil = dc.xception_shape(*case)
    x, w9, _ = operands((N, H, W, C, stride, pad, dil))
    y32 = aten_fprop(x, w9, stride, pad, dil).reshape(-1, C)
    rejects(lambda: dc.check_stats("unrounded", kernel_stats(y32), to_bf16(y32), dc.stat_chain_dw(y32.shape[0], C, SMS)),
            "statistics")


# ------------------------------------------------------------------------------------------------ entry-point refusal
@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU host only: the refusal returns before any CUDA call")
def test_entry_points_refuse_unaligned_channel_slices():
    """Every depthwise load and store is 16 bytes wide: a slice at a channel offset that is not a multiple of 8 (whose C
    and pitch are multiples of 8) must be refused, not launched."""
    from seg_b200 import lib
    if not os.path.exists(lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = lib.load()
    N, H, W, C = 1, 5, 5, 16
    buf = torch.zeros(N, H, W, C + 16, dtype=torch.bfloat16)
    ok, bad = buf[..., 8:8 + C], buf[..., 4:4 + C]
    assert ok.data_ptr() % 16 == 0 and bad.data_ptr() % 16 == 8
    d = lib.make_conv_desc(N, H, W, C, C, 3, 3, 1, 1, 1, ldx=C + 16, ldy=C + 16)
    w9 = torch.zeros(9, C)
    scratch = torch.zeros(int(L.seg_dwconv_scratch_floats(C)))
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    calls = {
        "fwd x": lambda: L.seg_dwconv3x3_fwd(ctypes.byref(d), p(bad), p(w9), p(ok), None, None, None, None),
        "fwd y": lambda: L.seg_dwconv3x3_fwd(ctypes.byref(d), p(ok), p(w9), p(bad), None, None, None, None),
        "bwd_data dy": lambda: L.seg_dwconv3x3_bwd_data(ctypes.byref(d), p(bad), p(w9), p(ok), 0.0, None),
        "bwd_data dx": lambda: L.seg_dwconv3x3_bwd_data(ctypes.byref(d), p(ok), p(w9), p(bad), 0.0, None),
        "bwd_weight dy": lambda: L.seg_dwconv3x3_bwd_weight(ctypes.byref(d), p(bad), p(ok), p(w9), 0.0, p(scratch), None),
        "bwd_weight x": lambda: L.seg_dwconv3x3_bwd_weight(ctypes.byref(d), p(ok), p(bad), p(w9), 0.0, p(scratch), None),
    }
    for what, fn in calls.items():
        assert fn() == 1, what
        assert "16-byte aligned" in lib.last_error(), (what, lib.last_error())
