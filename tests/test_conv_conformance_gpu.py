"""Conformance sweep of the convolution kernels (fprop, dgrad, wgrad; wgmma and CUDA-core paths).

Every case is checked element by element against a float64 reference with the bound of tests/conv_check.py, written
into guarded buffers (sentinel guard channels on both sides of the slice and a trailing guard image, which must come back
bit for bit; the logical region starts as the sentinel whenever beta = 0, so an element the kernel never wrote is caught),
and run twice: the wgmma results must be bit-identical between the runs.  Each case appends its bound usage to
gpu_out_dir/conv_conformance.txt.

The schedule cases are sized from the SM count at run time: the persistent fprop / dgrad grid is min(tiles, SMs) CTAs
and CTA b runs tiles b, b + grid, ..., so 1, 2, SMs - 1, SMs, SMs + 1, 2 SMs + 1, 3 SMs + 2 and 8 SMs + 3 tiles give one
idle consumer, one CTA with two tiles, odd tile counts per CTA and the producer running several tiles ahead of the
consumers (1 k-block per tile), with 1, 5 and 9 k-blocks per tile against rings of 4 and 6 stages."""
import ctypes
import math
import os

import pytest
import torch

import conv_check as cc

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import lib, ops
    from seg_b200.lib import IMPL_AUTO, IMPL_SIMT, IMPL_TC
else:  # keep collection working without a GPU
    IMPL_AUTO, IMPL_SIMT, IMPL_TC = 0, 1, 2

DEV = "cuda"
NAMES = {IMPL_AUTO: "auto", IMPL_SIMT: "simt", IMPL_TC: "tc"}
BF16, F32 = torch.bfloat16, torch.float32


def outsz(H, R, stride, pad, dil):
    return (H + 2 * pad - dil * (R - 1) - 1) // stride + 1


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def log(gpu_out_dir):
    f = open(os.path.join(gpu_out_dir, "conv_conformance.txt"), "a")

    def write(line):
        f.write(line + "\n")
        f.flush()

    yield write
    f.close()


def place(t, lead=None):
    """A bf16 NHWC device tensor holding t: dense, or a channel slice at offset `lead` of a wider buffer whose pitch is
    a multiple of 8 and whose other channels hold the sentinel (a kernel reading outside the slice produces NaNs)."""
    if lead is None:
        return t.to(DEV, BF16).contiguous()
    N, H, W, C = t.shape
    trail = cc.GUARD + (-(lead + C + cc.GUARD)) % 8
    buf = cc.sentinel_fill(torch.empty(N, H, W, lead + C + trail, dtype=BF16, device=DEV))
    buf[..., lead:lead + C] = t.to(DEV, BF16)
    return buf[..., lead:lead + C]


def fmt(u):
    return f"{u:.4f}"


# ------------------------------------------------------------------------------------------------ runners
def run_fprop(log, case, x, w, stride=1, pad=0, dil=1, impl=IMPL_TC, out_dtype=BF16, bias=None, beta=0.0, stats=False,
              lead=cc.GUARD, trail=cc.GUARD, x_lead=None, seed=0, note=""):
    N, H, W, C = x.shape
    K, _, R, S = w.shape
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, S, stride, pad, dil)
    old = None
    if beta != 0.0:
        old = cc.make_x(N, P, Q, K, seed + 100)
        if out_dtype == F32:
            old = old + torch.randn(old.shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 2 ** -12
            old = old.float().double()
    r = cc.fprop_ref(x, w, stride, pad, dil, bias=bias, beta=beta, old=old)
    xin = place(x, x_lead)
    wp = ops.pack_weight(w.float().to(DEV))
    bias_d = bias.float().to(DEV) if bias is not None else None
    runs = []
    for _ in range(2):
        g = cc.Guarded(N, P, Q, K, out_dtype, lead, trail, device=DEV)
        if old is not None:
            g.view.copy_(old.to(DEV, out_dtype))
        st = ops.new_stats(K, DEV) if stats else None
        ops.conv2d_fwd(xin, wp, K, R, S, stride, pad, dil, out=g.view, bias=bias_d, beta=beta, stats=st, impl=impl)
        torch.cuda.synchronize()
        cc.check_guards(case, g.buf, g.guard_mask())
        cc.check_written(case, g.view)
        runs.append((g.view.clone(), st))
    y, st = runs[0]
    out_bf16 = out_dtype == BF16
    usage = cc.check_elements(case, y, r, out_bf16, staged=out_bf16 and beta != 0.0 and impl != IMPL_SIMT)
    su = None
    if stats:
        M = N * P * Q
        chain = {IMPL_SIMT: cc.stat_chain_simt(M, K, sms()), IMPL_TC: cc.stat_chain_tc(K)}.get(
            impl, max(cc.stat_chain_simt(M, K, sms()), cc.stat_chain_tc(K)))  # AUTO: either path
        su = cc.check_stats(case, st, y.reshape(M, K), chain)
    if impl == IMPL_TC:
        assert torch.equal(runs[0][0].view(torch.int16 if out_bf16 else torch.int32),
                           runs[1][0].view(torch.int16 if out_bf16 else torch.int32)), f"{case}: output not bit-reproducible"
        if stats:
            assert torch.equal(runs[0][1], runs[1][1]), f"{case}: statistics not bit-reproducible"
    log(f"fprop {NAMES[impl]} {case} n={r.n} usage={fmt(usage)}" + (f" stats_usage={fmt(su)}" if stats else "") + note)
    return y, st


def run_dgrad(log, case, dy, w, x_shape, stride=1, pad=0, dil=1, impl=IMPL_TC, beta=0.0, lead=cc.GUARD, dy_lead=None,
              seed=0, note=""):
    """dx pitch rounded up to a multiple of 8 (a requirement of the wgmma path's supported()): with lead = 3 the slice
    still starts off a 16-byte boundary, which takes the epilogue's scalar stores."""
    N, H, W, C = x_shape
    trail = cc.GUARD + (-(lead + C + cc.GUARD)) % 8
    K, _, R, S = w.shape
    old = cc.make_x(N, H, W, C, seed + 200) if beta != 0.0 else None
    r = cc.dgrad_ref(dy, w, x_shape, stride, pad, dil, beta=beta, old=old)
    dyin = place(dy, dy_lead)
    wp = ops.pack_weight(w.float().to(DEV))
    runs = []
    for _ in range(2):
        g = cc.Guarded(N, H, W, C, BF16, lead, trail, device=DEV)
        if old is not None:
            g.view.copy_(old.to(DEV, BF16))
        ops.conv2d_dgrad(dyin, wp, x_shape, R, S, stride, pad, dil, out=g.view, beta=beta, impl=impl)
        torch.cuda.synchronize()
        cc.check_guards(case, g.buf, g.guard_mask())
        cc.check_written(case, g.view)
        runs.append(g.view.clone())
    usage = cc.check_elements(case, runs[0], r, True, staged=beta != 0.0 and impl != IMPL_SIMT)
    if impl == IMPL_TC:
        assert torch.equal(runs[0].view(torch.int16), runs[1].view(torch.int16)), f"{case}: output not bit-reproducible"
    log(f"dgrad {NAMES[impl]} {case} n={r.n} usage={fmt(usage)}" + note)
    return runs[0], r


def wgrad_plan(N, P, Q, K, C, R, S):
    """(BN, splits, k-blocks per split) of the wgmma wgrad (mirror of seg_conv_tc.cu's wgrad_plan)."""
    wide = R * S >= 9 and C >= 256 and C % 256 == 0
    bn = 64 if C <= 64 else (256 if wide else 128)
    kbt = -(-N * P * Q // 64)
    tiles = -(-K // 128) * -(-C // bn) * R * S
    splits = min(max(1, sms() // tiles), kbt, 1024)
    kps = -(-kbt // splits)
    return bn, -(-kbt // kps), kps


def run_wgrad(log, case, dy, x, R, S, stride=1, pad=0, dil=1, impl=IMPL_TC, lead=cc.GUARD, dy_lead=None, x_lead=None,
              seed=0, note=""):
    """Through the C ABI so that the split-K workspace can start as NaN: every element of every split's slice must be
    written before the reduction reads it.  dw starts as random values: the result must be dw_old + grad."""
    N, H, W, C = x.shape
    K = dy.shape[-1]
    assert N * dy.shape[1] * dy.shape[2] <= cc.LARGEST_WGRAD_PIXELS
    dw_old = torch.randn(R * S, K, C, generator=torch.Generator().manual_seed(seed + 300)).double()
    r = cc.wgrad_ref(dy, x, R, S, stride, pad, dil, old=dw_old)
    dyin, xin = place(dy, dy_lead), place(x, x_lead)
    d = lib.make_conv_desc(N, H, W, C, K, R, S, stride, pad, dil, ldx=ops.ld(xin), ldy=ops.ld(dyin))
    nws = int(lib.load().seg_conv2d_wgrad_workspace_floats(ctypes.byref(d), impl))
    assert nws >= 0
    splits = nws // (R * S * K * C) if nws else 1
    runs = []
    for _ in range(2):
        f = cc.FlatGuarded((R * S, K, C), F32, lead=lead, device=DEV)
        f.view.copy_(dw_old.float())
        ws = torch.full((nws,), float("nan"), device=DEV) if nws else None
        lib.call("seg_conv2d_wgrad", ctypes.byref(d), lib.ptr(dyin), lib.ptr(xin), lib.ptr(f.view), lib.ptr(ws), impl)
        torch.cuda.synchronize()
        cc.check_guards(case, f.buf, f.guard_mask())
        runs.append(f.view.clone())
    usage = cc.check_elements(case, runs[0], r, False, splits=splits if impl != IMPL_SIMT else 0)
    if impl == IMPL_TC:
        assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), f"{case}: dW not bit-reproducible"
    log(f"wgrad {NAMES[impl]} {case} n={r.n} splits={splits} usage={fmt(usage)}" + note)
    return runs[0], splits


# ------------------------------------------------------------------------------------------------ 1. schedule
def shape_for_row_tiles(t):
    """(N, H, W) with ceil(N H W / 128) == t, M not a multiple of 128 where possible (a row tail in the last tile)."""
    lo, hi = (t - 1) * cc.BM + (1 if t > 1 else 100), t * cc.BM
    for N in (1, 2, 3, 4):
        h0 = max(2, math.isqrt(max(lo // N, 1)))
        for H in range(h0, h0 + 400):
            W = -(-lo // (N * H))
            if W >= 2 and N * H * W <= hi:
                return N, H, W
    raise AssertionError(f"no map with {t} row tiles")


def schedule_counts():
    s = sms()
    return [1, 2, s - 1, s, s + 1, 2 * s + 1, 3 * s + 2, 8 * s + 3]


KB_OPTIONS = {1: (1, 64), 5: (1, 320), 9: (3, 64)}  # k-blocks per tile -> (R, contraction channels)
KB_FOR_COUNT = [9, 5, 1, 9, 5, 1, 9, 1]             # the 8 * SMs + 3 count takes the 1-k-block tiles: the cheap reference


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("ci", range(8), ids=["1", "2", "sms-1", "sms", "sms+1", "2sms+1", "3sms+2", "8sms+3"])
def test_schedule_fprop(log, ci, bn):
    count = schedule_counts()[ci]
    kb = KB_FOR_COUNT[ci]
    R, C = KB_OPTIONS[kb]
    out_dtype = F32 if (bn == 64 and ci % 2) else BF16
    K = 128 if bn == 128 else (48 if out_dtype == F32 else 64)
    N, H, W = shape_for_row_tiles(count)
    M = N * H * W
    tiles = -(-M // cc.BM) * -(-K // bn)
    assert tiles == count
    assert (K <= 64 or out_dtype == F32) == (bn == 64)
    assert (-(-C // 64)) * R * R == kb
    x, w = cc.make_x(N, H, W, C, ci), cc.make_w(K, C, R, R, ci + 50)
    grid = min(tiles, sms())
    run_fprop(log, f"sched bn={bn} tiles={tiles} kb={kb} {N}x{H}x{W}x{C}->{K}", x, w, 1, R // 2, 1, out_dtype=out_dtype,
              stats=True, seed=ci, note=f" grid={grid} tiles_per_cta={tiles / grid:.2f}")


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("ci", range(8), ids=["1", "2", "sms-1", "sms", "sms+1", "2sms+1", "3sms+2", "8sms+3"])
def test_schedule_dgrad(log, ci, bn):
    count = schedule_counts()[ci]
    kb = KB_FOR_COUNT[ci]
    R, K = KB_OPTIONS[kb]
    C = bn
    N, H, W = shape_for_row_tiles(count)
    tiles = -(-N * H * W // cc.BM) * -(-C // bn)
    assert tiles == count
    dy, w = cc.make_x(N, H, W, K, ci + 7), cc.make_w(K, C, R, R, ci + 60)
    grid = min(tiles, sms())
    run_dgrad(log, f"sched bn={bn} tiles={tiles} kb={kb} {N}x{H}x{W}x{C}<-{K}", dy, w, (N, H, W, C), 1, R // 2, 1,
              seed=ci, note=f" grid={grid} tiles_per_cta={tiles / grid:.2f}")


@pytest.mark.parametrize("beta", [0.0, 0.5])
def test_schedule_dgrad_unreachable_classes_many_tiles(log, beta):
    """1x1 stride-2 dgrad on a large map: three of the four parity classes get no tap, each ~8 tiles per CTA of the
    zero-iteration kernel (zeros over the sentinel, or beta * old)."""
    N, H, W, C, K = 8, 256, 256, 16, 16
    dy, w = cc.make_x(N, 128, 128, K, 1), cc.make_w(K, C, 1, 1, 2)
    tiles = -(-N * 128 * 128 // cc.BM)
    dx, _ = run_dgrad(log, f"s2 1x1 unreachable classes beta={beta} {N}x{H}x{W}x{C}", dy, w, (N, H, W, C), 2, 0, 1,
                      beta=beta, seed=3, note=f" tiles_per_class={tiles} tiles_per_cta={tiles / min(tiles, sms()):.2f}")
    if beta == 0.0:
        assert dx[:, 1::2].abs().max().item() == 0 and dx[:, :, 1::2].abs().max().item() == 0


# ------------------------------------------------------------------------------------------------ 2. tails and geometry
# name: (N, H, W, C, K, R, stride, pad, dil)
GEOMETRY = {
    "m1": (1, 1, 1, 64, 64, 1, 1, 0, 1),
    "m2_image_pool": (2, 1, 1, 320, 256, 1, 1, 0, 1),
    "m127": (1, 1, 127, 64, 72, 1, 1, 0, 1),
    "m128": (1, 8, 16, 64, 24, 1, 1, 0, 1),
    "m129": (1, 3, 43, 72, 64, 1, 1, 0, 1),
    "c8_k8_3x3_pad0": (2, 9, 9, 8, 8, 3, 1, 0, 1),
    "c200_k19_1x1": (2, 7, 9, 200, 19, 1, 1, 0, 1),
    "c56_k24_3x3_pad2": (1, 7, 8, 56, 24, 3, 1, 2, 1),
    "c304_k48_3x3": (1, 9, 9, 304, 48, 3, 1, 1, 1),
    "c72_k72_3x3_s2_odd": (1, 17, 17, 72, 72, 3, 2, 1, 1),
    "c56_k136_3x3_s2_even": (2, 16, 16, 56, 136, 3, 2, 1, 1),
    "c200_k200_1x1_s2": (2, 13, 13, 200, 200, 1, 2, 0, 1),
    "c64_k64_3x3_s2_dil2": (1, 15, 15, 64, 64, 3, 2, 2, 2),
    "c64_k48_3x3_s3": (1, 14, 14, 64, 48, 3, 3, 1, 1),
    "c16_k24_5x5": (1, 12, 12, 16, 24, 5, 1, 2, 1),
    "c16_k32_7x7": (1, 15, 15, 16, 32, 7, 1, 3, 1),
    "c16_k8_dil18": (1, 33, 33, 16, 8, 3, 1, 18, 18),
}
GEO_IDS = list(GEOMETRY)
IMPLS = pytest.mark.parametrize("impl", [IMPL_SIMT, IMPL_TC], ids=["simt", "tc"])


@IMPLS
@pytest.mark.parametrize("name", GEO_IDS)
def test_geometry_fprop(log, name, impl):
    N, H, W, C, K, R, stride, pad, dil = GEOMETRY[name]
    x, w = cc.make_x(N, H, W, C, 11), cc.make_w(K, C, R, R, 12)
    bias = torch.randn(K, generator=torch.Generator().manual_seed(13)).double()
    assert C * R * R <= cc.LARGEST_FPROP_F32_N
    stats = K % 8 == 0
    y, st = run_fprop(log, f"{name} bf16 aligned", x, w, stride, pad, dil, impl=impl, bias=bias, stats=stats)
    run_fprop(log, f"{name} bf16 unaligned x-slice", x, w, stride, pad, dil, impl=impl, lead=3, x_lead=8)
    # fp32 output; K = 19 also dense with pitch 19
    dense = K % 4 != 0
    run_fprop(log, f"{name} fp32" + (" dense" if dense else " unaligned"), x, w, stride, pad, dil, impl=impl,
              out_dtype=F32, bias=bias, stats=impl == IMPL_TC, lead=0 if dense else 1, trail=0 if dense else cc.GUARD)
    if stats and impl == IMPL_TC:  # the statistics do not depend on where the output lives
        _, st_dense = run_fprop(log, f"{name} bf16 dense", x, w, stride, pad, dil, impl=impl, bias=bias, stats=True,
                                lead=0, trail=0)
        assert torch.equal(st, st_dense), f"{name}: statistics differ between a dense and a guarded output"


@IMPLS
@pytest.mark.parametrize("name", GEO_IDS)
def test_geometry_dgrad(log, name, impl):
    N, H, W, C, K, R, stride, pad, dil = GEOMETRY[name]
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, R, stride, pad, dil)
    dy, w = cc.make_x(N, P, Q, K, 21), cc.make_w(K, C, R, R, 22)
    # K = 19: dy lives in a slice whose pitch is a multiple of 8, as the wgmma path needs
    run_dgrad(log, f"{name} aligned", dy, w, (N, H, W, C), stride, pad, dil, impl=impl, dy_lead=8 if K % 8 else None)
    run_dgrad(log, f"{name} unaligned dy-slice", dy, w, (N, H, W, C), stride, pad, dil, impl=impl, lead=3, dy_lead=8)


@IMPLS
@pytest.mark.parametrize("name", GEO_IDS)
def test_geometry_wgrad(log, name, impl):
    N, H, W, C, K, R, stride, pad, dil = GEOMETRY[name]
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, R, stride, pad, dil)
    x, dy = cc.make_x(N, H, W, C, 31), cc.make_x(N, P, Q, K, 32)
    # K = 19: dy lives in a slice whose pitch is a multiple of 8, as the wgmma path needs
    dy_lead = 8 if K % 8 else None
    run_wgrad(log, f"{name} aligned", dy, x, R, R, stride, pad, dil, impl=impl, dy_lead=dy_lead)
    run_wgrad(log, f"{name} unaligned dw, slices", dy, x, R, R, stride, pad, dil, impl=impl, lead=1, dy_lead=8, x_lead=8)


# the limits of tc::supported(): the im2col corners are signed 8-bit, |dil (R - 1) - pad| <= 127 and pad <= 127
EDGES = {
    "pad127_1x1": (1, 1, 1, 8, 8, 1, 1, 127, 1),       # pad = 127 and dil (R - 1) - pad = -127
    "dil64_pad1_3x3": (1, 130, 130, 8, 8, 3, 1, 1, 64),  # dil (R - 1) - pad = +127
}
PAST_EDGES = {
    "pad128_1x1": (1, 1, 1, 8, 8, 1, 1, 128, 1),
    "dil64_pad0_3x3": (1, 131, 131, 8, 8, 3, 1, 0, 64),  # dil (R - 1) - pad = 128
}


@pytest.mark.parametrize("name", list(EDGES))
def test_supported_edges_run_on_tc(log, name):
    N, H, W, C, K, R, stride, pad, dil = EDGES[name]
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, R, stride, pad, dil)
    x, w = cc.make_x(N, H, W, C, 41), cc.make_w(K, C, R, R, 42)
    dy = cc.make_x(N, P, Q, K, 43)
    run_fprop(log, f"edge {name}", x, w, stride, pad, dil, impl=IMPL_TC, stats=True)
    run_dgrad(log, f"edge {name}", dy, w, (N, H, W, C), stride, pad, dil, impl=IMPL_TC)
    if R > 1:  # the 1x1 pad-127 wgrad would contract over 65025 pixels, all but one of them padding
        run_wgrad(log, f"edge {name}", dy, x, R, R, stride, pad, dil, impl=IMPL_TC)


@pytest.mark.parametrize("name", list(PAST_EDGES))
def test_past_supported_edges_auto_falls_back(log, name):
    N, H, W, C, K, R, stride, pad, dil = PAST_EDGES[name]
    P, Q = outsz(H, R, stride, pad, dil), outsz(W, R, stride, pad, dil)
    x, w = cc.make_x(N, H, W, C, 51), cc.make_w(K, C, R, R, 52)
    dy = cc.make_x(N, P, Q, K, 53)
    run_fprop(log, f"past edge {name}", x, w, stride, pad, dil, impl=IMPL_AUTO, stats=True)
    run_dgrad(log, f"past edge {name}", dy, w, (N, H, W, C), stride, pad, dil, impl=IMPL_AUTO)
    if R > 1:
        run_wgrad(log, f"past edge {name}", dy, x, R, R, stride, pad, dil, impl=IMPL_AUTO)
    wp = ops.pack_weight(w.float().to(DEV))
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.conv2d_fwd(place(x), wp, K, R, R, stride, pad, dil, impl=IMPL_TC)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.conv2d_dgrad(place(dy), wp, (N, H, W, C), R, R, stride, pad, dil, impl=IMPL_TC)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.conv2d_wgrad(place(dy), place(x), R, R, stride, pad, dil, impl=IMPL_TC)


# im2col maps of tensors under 128 KiB take a driver workaround (make_map_im2col): just under, at and just over it
IM2COL_SIZES = {
    "128KiB-16B": (1, 1, 8191, 8),   # 8191 pixels x 8 channels x 2 B
    "128KiB": (1, 32, 32, 64),
    "128KiB+row": (1, 33, 32, 64),
}


@pytest.mark.parametrize("name", list(IM2COL_SIZES))
def test_im2col_small_tensor_boundary(log, name):
    N, H, W, C = IM2COL_SIZES[name]
    nbytes = N * H * W * C * 2
    assert nbytes == {"128KiB-16B": 131056, "128KiB": 131072, "128KiB+row": 131072 + W * C * 2}[name]
    K = C
    x, w = cc.make_x(N, H, W, C, 61), cc.make_w(K, C, 3, 3, 62)
    run_fprop(log, f"im2col {name}", x, w, 1, 1, 1, impl=IMPL_TC, stats=True)
    dy = cc.make_x(N, H, W, K, 63)  # 3x3 pad 1: dy has the same size, read through the same kind of map
    run_dgrad(log, f"im2col {name}", dy, w, (N, H, W, C), 1, 1, 1, impl=IMPL_TC)
    run_wgrad(log, f"im2col {name}", dy, x, 3, 3, 1, 1, 1, impl=IMPL_TC)


# ------------------------------------------------------------------------------------------------ 3. beta, slices
@IMPLS
@pytest.mark.parametrize("out_dtype", [BF16, F32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("beta", [0.0, 1.0, 0.5])
def test_fprop_beta(log, beta, out_dtype, impl):
    N, H, W, C, K = 2, 9, 11, 64, 48
    x, w = cc.make_x(N, H, W, C, 71), cc.make_w(K, C, 3, 3, 72)
    bias = torch.randn(K, generator=torch.Generator().manual_seed(73)).double()
    for lead in (cc.GUARD, 3):
        run_fprop(log, f"beta={beta} {'bf16' if out_dtype == BF16 else 'fp32'} lead={lead}", x, w, 1, 1, 1, impl=impl,
                  out_dtype=out_dtype, bias=bias, beta=beta, lead=lead, seed=int(beta * 10))


@IMPLS
@pytest.mark.parametrize("geom", ["3x3_s1", "3x3_s2", "1x1_s2"])
@pytest.mark.parametrize("beta", [0.0, 1.0, 0.5])
def test_dgrad_beta(log, beta, geom, impl):
    """With stride 2 and a 1x1 filter three parity classes get no tap: zeros over the sentinel for beta = 0, the old
    values for beta = 1 and 0.5 * old for beta = 0.5."""
    R, stride, pad = {"3x3_s1": (3, 1, 1), "3x3_s2": (3, 2, 1), "1x1_s2": (1, 2, 0)}[geom]
    N, H, W, C, K = 2, 13, 13, 64, 48
    P, Q = outsz(H, R, stride, pad, 1), outsz(W, R, stride, pad, 1)
    dy, w = cc.make_x(N, P, Q, K, 81), cc.make_w(K, C, R, R, 82)
    for lead in (cc.GUARD, 3):
        run_dgrad(log, f"beta={beta} {geom} lead={lead}", dy, w, (N, H, W, C), stride, pad, 1, impl=impl, beta=beta,
                  lead=lead, dy_lead=8, seed=int(beta * 10))


def test_unaligned_input_slice_auto_falls_back_tc_raises(log):
    """An operand slice at channel offset 4 (8 bytes: not 16-byte aligned, so no TMA map) with a pitch that is a
    multiple of 8: AUTO must run it on the CUDA cores and get it right; IMPL_TC must refuse it."""
    N, H, W, C, K = 2, 9, 9, 64, 64
    x, w = cc.make_x(N, H, W, C, 91), cc.make_w(K, C, 3, 3, 92)
    dy = cc.make_x(N, H, W, K, 93)
    run_fprop(log, "x at channel offset 4", x, w, 1, 1, 1, impl=IMPL_AUTO, x_lead=4, stats=True)
    run_dgrad(log, "dy at channel offset 4", dy, w, (N, H, W, C), 1, 1, 1, impl=IMPL_AUTO, dy_lead=4)
    run_wgrad(log, "dy at channel offset 4", dy, x, 3, 3, 1, 1, 1, impl=IMPL_AUTO, dy_lead=4)
    run_wgrad(log, "x at channel offset 4", dy, x, 3, 3, 1, 1, 1, impl=IMPL_AUTO, x_lead=4)
    xs, dys = place(x, 4), place(dy, 4)
    assert ops.ld(xs) % 8 == 0 and xs.data_ptr() % 16 == 8
    wp = ops.pack_weight(w.float().to(DEV))
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.conv2d_fwd(xs, wp, K, 3, 3, 1, 1, 1, impl=IMPL_TC)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.conv2d_dgrad(dys, wp, (N, H, W, C), 3, 3, 1, 1, 1, impl=IMPL_TC)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.conv2d_wgrad(dys, place(x), 3, 3, 1, 1, 1, impl=IMPL_TC)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.conv2d_wgrad(place(dy), xs, 3, 3, 1, 1, 1, impl=IMPL_TC)


@IMPLS
def test_fprop_statistics_with_beta_is_rejected(impl):
    N, H, W, C, K = 1, 5, 5, 64, 64
    x, w = cc.make_x(N, H, W, C, 95), cc.make_w(K, C, 1, 1, 96)
    y = torch.zeros(N, H, W, K, dtype=BF16, device=DEV)
    with pytest.raises(RuntimeError, match="beta = 0"):
        ops.conv2d_fwd(place(x), ops.pack_weight(w.float().to(DEV)), K, 1, 1, out=y, beta=0.5, stats=ops.new_stats(K, DEV),
                       impl=impl)


# ------------------------------------------------------------------------------------------------ 4. wgrad plans
def pixels_for_kblocks(kb):
    """(N, H, W) of a 1x1 stride-1 map with exactly kb 64-pixel k-blocks."""
    lo, hi = (kb - 1) * 64 + 1, kb * 64
    for H in range(max(2, math.isqrt(lo)), 1000):
        W = -(-lo // H)
        if H * W <= hi:
            return 1, H, W
    raise AssertionError(kb)


WGRAD_PLANS = ["one_split", "many_splits", "capped_by_kblocks", "recounted", "bn256", "bn128_k512"]


@pytest.mark.parametrize("plan", WGRAD_PLANS)
def test_wgrad_plans(log, plan):
    s = sms()
    if plan == "one_split":  # tiles = 4 x 4 x 9 = 144 >= SMs
        N, H, W, C, K, R = 1, 9, 9, 448, 512, 3
    elif plan == "many_splits":  # one tile, 2 SMs k-blocks: SMs splits of 2
        (N, H, W), C, K, R = pixels_for_kblocks(2 * s), 64, 48, 1
    elif plan == "capped_by_kblocks":  # tiny M: 5 k-blocks, 5 splits
        N, H, W, C, K, R = 1, 15, 20, 64, 48, 1
    elif plan == "recounted":  # SMs + 1 k-blocks: 2 per split, so the split count is recounted to ceil((SMs + 1) / 2)
        (N, H, W), C, K, R = pixels_for_kblocks(s + 1), 64, 19, 1
    elif plan == "bn256":
        N, H, W, C, K, R = 1, 9, 9, 256, 48, 3
    else:
        N, H, W, C, K, R = 2, 20, 20, 128, 512, 1
    pad = R // 2
    bn, splits, kps = wgrad_plan(N, H, W, K, C, R, R)
    kbt = -(-N * H * W // 64)
    expect = {"one_split": lambda: splits == 1,
              "many_splits": lambda: splits == s and kps == 2,
              "capped_by_kblocks": lambda: splits == kbt == 5,
              "recounted": lambda: kps == 2 and splits == -(-(s + 1) // 2) and splits < s,
              "bn256": lambda: bn == 256 and splits > 1,
              "bn128_k512": lambda: bn == 128 and splits > 1}[plan]
    assert expect(), (plan, bn, splits, kps, kbt)
    x, dy = cc.make_x(N, H, W, C, 101), cc.make_x(N, H, W, K, 102)
    dy_lead = 8 if K % 8 else None
    for lead in (cc.GUARD, 1):
        _, got_splits = run_wgrad(log, f"plan {plan} lead={lead} {N}x{H}x{W}x{C}->{K} {R}x{R}", dy, x, R, R, 1, pad, 1,
                                  lead=lead, dy_lead=dy_lead, note=f" bn={bn} kblocks={kbt} per_split={kps}")
        assert got_splits == splits
