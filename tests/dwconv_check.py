"""Per-element conformance checker for the depthwise 3x3 kernels of seg_dwconv.cu: forward (+ BatchNorm statistics),
data gradient, weight gradient, and the [C][1][3][3] <-> [9][C] weight packing.

Pure torch on the CPU, like conv_check.py, whose guarded buffers, sentinels, statistics check and operand makers it
reuses (and elementwise_check.py's per-element check with explicit allowances): its own tests run without a GPU
(test_dwconv_check_cpu.py) and the GPU sweep (test_dwconv_conformance_gpu.py) feeds it what the kernels wrote.

Reference: the float64 grouped convolution (groups = C) of the bf16-exact activations with the fp32 taps (the kernels
keep the taps in registers as fp32; they are never rounded to bf16).  Magnitude T: the same operation on |operands|,
plus |beta old| where an old value is added.  Per-element bound (u32 = 2^-24, u_bf16 = 2^-8):

    |got - ref| <= r + e,   e = k u32 T                  (k: the fp32 roundings of the kernel's arithmetic, derived below)
                            r = u_bf16 (|ref| + e)       (bf16 outputs: the fp32 value, within e of ref, is rounded once)

"Bound usage" means what it means in conv_check: (|got - ref| - r)+ / e; an element fails above 1 and a case reports
its largest usage.  The grid mirror (dw_grid) copies seg_dwconv.cu's host function, so the weight gradient and the
statistics are charged the fp32 chains of the grid that is actually launched.
"""
import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

from conv_check import (GUARD, U32, UBF, FlatGuarded, Guarded, bf16_round, channel_scales, check_guards,  # noqa: F401
                        check_stats, check_written, is_sentinel, make_x, nchw, nhwc, sentinel_fill)
from elementwise_check import Bound, bound, check, check_exact  # noqa: F401

# Forward: o starts at 0 and takes one fmaf per tap in range, at most 9; each rounds once, by at most u32 times a partial
# sum, which is at most T.  Hence 9 u32 T before the single bf16 rounding (pack8).
K_FPROP = 9
# Data gradient: the same 9-long fma chain, then o += beta * old: the product and the sum round once each (or once when
# the compiler contracts them into an fma), by at most u32 T with T = |taps| |dy| + |beta old|.  No staged rounding: the
# convolution stays fp32 until the one bf16 rounding of the sum.
K_DGRAD = 9 + 2
# Weight gradient on top of the fp32 chain of wgrad_chain(): the fp64 total is rounded to fp32 (1), then
# dw9 = beta * dw9 + v: product and sum (2).  The chain itself already counts the rounding to fp32.
K_WGRAD_BETA = 2
# dw_unpack_wgrad: g = beta * g + v (product and sum; exact copies when beta = 0).
K_UNPACK = 2
# The longest fp32 chain and the largest pixel count of the GPU sweep's weight-gradient cases (which asserts every case
# stays within both): the bound grows with both, and the checker's self-tests show that one dropped pixel is still
# caught when they are reached together.
LARGEST_DW_WGRAD_CHAIN = 300
LARGEST_DW_WGRAD_PIXELS = 300_000

NAMES_NHWC = ("n", "h", "w", "c")
NAMES_W9 = ("tap", "c")
DW_WGRAD_BLOCKS_PER_SM = 4   # seg_dwconv.cu: the weight gradient's cap
DW_BLOCKS_PER_SM = 6         # the forward's and the data gradient's cap


def outsz(H, stride, pad, dil):
    return (H + 2 * pad - 2 * dil - 1) // stride + 1


# The Aligned-Xception layers of the GPU sweep, scaled down: the backbone's channel counts, strides and dilations, with
# "same" padding (pad = dil if dil > 1 else 1, as SeparableConv2d does) on small maps of both parities.
XCEPTION_C = (64, 128, 256, 728, 1024, 1536)
XCEPTION_CASES = [(C, stride, dil) for C in XCEPTION_C for stride in (1, 2) for dil in (1, 2, 4)]


def xception_shape(C, stride, dil):
    """(N, H, W, C, stride, pad, dil) of one scaled-down Xception layer."""
    return 2, 11 + stride, 9 + dil, C, stride, dil if dil > 1 else 1, dil


# ------------------------------------------------------------------------------------------------ grid mirror
def dw_grid(M, C, sms, blocks_per_sm=DW_BLOCKS_PER_SM):
    """(gx, gy, rows_par) of a depthwise launch over M rows (mirror of seg_dwconv.cu's dw_grid and dw_map): a block of
    256 threads covers GB = min(C / 8, 256) channel groups and rows_par = 256 / GB rows at a time; gy blocks span the
    channels, and gx, two rows per thread at most, is capped at sms * blocks_per_sm blocks in all."""
    G = C // 8
    GB = min(G, 256)
    rows_par = 256 // GB
    gy = -(-G // GB)
    gx = -(-M // (rows_par * 2))
    cap = (sms * blocks_per_sm + gy - 1) // gy
    return max(1, min(gx, cap)), gy, rows_par


def rows_per_thread(M, C, sms, blocks_per_sm):
    gx, _, rows_par = dw_grid(M, C, sms, blocks_per_sm)
    return -(-M // (gx * rows_par))


def stat_chain_dw(M, C, sms):
    """Longest fp32 chain of the forward's statistics: every thread sums its grid-strided rows, then the block adds its
    rows_par row lanes; the fp64 atomics are exact and the totals stay fp64.  The + 1 covers the rounding of o * o in
    the sum of squares (at most u32 times the sum of squares)."""
    gx, _, rows_par = dw_grid(M, C, sms, DW_BLOCKS_PER_SM)
    return -(-M // (gx * rows_par)) + rows_par + 1


def wgrad_chain(M, C, sms):
    """Longest fp32 chain of the weight gradient: one fma per row a thread visits, the block reduction over rows_par row
    lanes, the exact fp64 sum of the block partials, and one rounding of that total to fp32."""
    gx, _, rows_par = dw_grid(M, C, sms, DW_WGRAD_BLOCKS_PER_SM)
    return -(-M // (gx * rows_par)) + rows_par + 1


# ------------------------------------------------------------------------------------------------ operands
def make_w9(C, seed):
    """Packed fp32 taps [9][C] (fp32-exact float64; not bf16-exact, not symmetric) with per-channel magnitudes."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(9, C, generator=g, dtype=torch.float64) / 3 * channel_scales(C, seed + 1)
    return w.float().double()


def w9_to_oihw(w9):
    """[9][C] -> [C, 1, 3, 3] (tap t = 3 r + s)."""
    return w9.t().reshape(w9.shape[1], 1, 3, 3)


def oihw_to_w9(w):
    return w.reshape(w.shape[0], 9).t()


# ------------------------------------------------------------------------------------------------ references
def fprop_ref(x, w9, stride, pad, dil):
    """x: NHWC bf16-exact, w9: [9][C]; returns the Bound of y [N, P, Q, C] (bf16 output)."""
    C = x.shape[-1]
    xd, wd = nchw(x.double()), w9_to_oihw(w9.double())
    ref = nhwc(F.conv2d(xd, wd, None, stride, pad, dil, groups=C))
    mag = nhwc(F.conv2d(xd.abs(), wd.abs(), None, stride, pad, dil, groups=C))
    return bound(ref, K_FPROP * U32 * mag, True, NAMES_NHWC)


def dgrad_ref(dy, w9, x_shape, stride, pad, dil, beta=0.0, old=None):
    """dy: NHWC [N, P, Q, C]; returns the Bound of dx = beta old + dw^T(dy) [N, H, W, C] (bf16 output)."""
    N, H, W, C = x_shape
    dyd, wd = nchw(dy.double()), w9_to_oihw(w9.double())
    size = (N, C, H, W)
    ref = nhwc(nn_grad.conv2d_input(size, wd, dyd, stride, pad, dil, groups=C))
    mag = nhwc(nn_grad.conv2d_input(size, wd.abs(), dyd.abs(), stride, pad, dil, groups=C))
    if beta != 0.0:
        ref = ref + beta * old.double()
        mag = mag + (beta * old.double()).abs()
    return bound(ref, K_DGRAD * U32 * mag, True, NAMES_NHWC)


def wgrad_ref(dy, x, stride, pad, dil, chain, beta=0.0, old=None):
    """dy: NHWC [N, P, Q, C], x: NHWC [N, H, W, C]; returns the Bound of dw9 = beta old + sum dy x_shifted, [9][C] fp32;
    chain: wgrad_chain() of the launch."""
    C = x.shape[-1]
    dyd, xd = nchw(dy.double()), nchw(x.double())
    ref = oihw_to_w9(nn_grad.conv2d_weight(xd, (C, 1, 3, 3), dyd, stride, pad, dil, groups=C))
    mag = oihw_to_w9(nn_grad.conv2d_weight(xd.abs(), (C, 1, 3, 3), dyd.abs(), stride, pad, dil, groups=C))
    if beta != 0.0:
        ref = ref + beta * old.double()
        mag = mag + (beta * old.double()).abs()
    return bound(ref, (chain + K_WGRAD_BETA) * U32 * mag, False, NAMES_W9)


def unpack_ref(g9, beta=0.0, old=None):
    """dw_unpack_wgrad: g [C, 1, 3, 3] = beta old + g9 rearranged; fp32 output."""
    ref = w9_to_oihw(g9.double())
    mag = ref.abs()
    if beta != 0.0:
        ref = ref + beta * old.double()
        mag = mag + (beta * old.double()).abs()
    return bound(ref, K_UNPACK * U32 * mag, False, ("c", "one", "r", "s"))


def check_fprop(case, got, b):
    return check(case, "dwconv fwd", got, b)


def check_dgrad(case, got, b):
    return check(case, "dwconv bwd_data", got, b)


def check_wgrad(case, got, b):
    return check(case, "dwconv bwd_weight", got, b)


def check_unpack(case, got, b):
    return check(case, "dw_unpack_wgrad", got, b)


def check_pack(case, got_w9, w_c133):
    """dw_pack_weight is a permutation: bit-exact."""
    check_exact(case, "dw_pack_weight", got_w9, oihw_to_w9(w_c133.double()), NAMES_W9)
