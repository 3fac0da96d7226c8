"""Per-element conformance checker for the streaming kernels of seg_elementwise.cu: BatchNorm statistics, apply
(+residual, ReLU, dropout), backward (two-launch and cooperative), max pool, adaptive average pool, bilinear resize,
ReLU and axpby.

Pure torch on the CPU, like conv_check.py, whose guarded buffers, sentinels, statistics check and operand makers it
reuses: its own tests run without a GPU (test_elementwise_check_cpu.py) and the GPU sweep
(test_elementwise_conformance_gpu.py) feeds it what the kernels wrote.

Reference: the float64 operation of the bf16-exact operands.  Per-element bound (u32 = 2^-24, u_bf16 = 2^-8):

    |got - ref| <= r + e,   e = k u32 T + (propagated allowance of inputs the kernel computed itself, e.g. sums)
                            r = 0 (fp32 outputs);  u_bf16 (|ref| + e)  (bf16 outputs: the kernel rounds its fp32 value,
                                which lies within e of ref, once)

T bounds the magnitude of every fp32 intermediate of the element (it is the same expression on |operands|), and k counts
the fp32 roundings of the kernel's arithmetic; each operation below derives its k.  "Bound usage" means what it means
in conv_check: (|got - ref| - r)+ / e; an element fails above 1 and a case reports its largest usage.

The grid mirrors (colreduce_grid, rowmap_grid, reduce2_grid, fused_grid) copy seg_elementwise.cu's host functions: the
BatchNorm sums are charged the length of the longest fp32 summation chain the launched grid produces.
"""
import math

import torch
import torch.nn.functional as F

from conv_check import (GUARD, U32, UBF, FlatGuarded, Guarded, bf16_round, channel_scales, check_guards,  # noqa: F401
                        check_stats, check_written, is_sentinel, nchw, nhwc, sentinel_fill, stat_chain_simt)

# Roundings charged to one output of the BatchNorm apply kernel (training statistics), relative to
# T = |gamma| istd (|x| + |mean|) + |beta| + |res|:
#   istd: var -> fp32 (1/2), rsqrtf + one Newton step whose 3 products and 1 subtraction round (4), hence ~4.5 relative
#   sc = gamma istd: 1 more (5.5);  mean -> fp32: 1;  sh = fma(-mean, sc, beta): 1;  fma(x, sc, sh): 1;  + res: 1.
# The worst sum over T's terms is |mean||sc| (5.5 + 1 + 1 + 1 + 1 = 9.5), hence 10.
K_APPLY = 10
# The same with the coefficients given as fp32 scale/shift (bn_apply): fma(x, sc, sh) and + res.
K_APPLY_SS = 2
# Relative bound of the fp32 coefficients the BatchNorm kernels derive per channel: save = (mean, istd) and
# scale/shift (mean: one rounding; istd: the 4.5 above or, in bn_finalize / bn_eval_scale_shift, an fp64 sqrt or rsqrtf
# (2 ulp) rounded once; scale: one product more; shift: two operations more on |mean sc| + |beta|).
K_COEF = 8
# Roundings charged to dx of the BatchNorm backward relative to |A dz'| + |B| (|x| + |mean|) + |A s0| / M
# (A = gamma istd, B = A istd s1 / M): cB carries 5 (a, istd, s1, inv_count and inv_count's own rounding), cC 4 + the
# product and difference with cB mean (2), the two fmas 1 each, and dz' its keep scale (3): 10 covers the largest sum.
K_DX = 10
KEEP_ROUNDINGS = 3  # dz * fp32(1 / fp32(1 - p)): 1 - p, the division and the product round once each
MAXN = 24           # bilinear_bwd_kernel's fast path: at most this many outputs per input row / column
# Ceiling of the fp32 summation chains of the GPU sweep's BatchNorm sums (which asserts every case stays within it): the
# checker's self-tests show that one dropped row is still caught at this length, where the bound is widest.
LONGEST_SUM_CHAIN = 1024


# ------------------------------------------------------------------------------------------------ element checks
class Bound:
    """ref: float64 reference; rnd / acc: the rounding and accumulation allowances per element; names: coordinates."""

    def __init__(self, ref, rnd, acc, names):
        self.ref, self.rnd, self.acc, self.names = ref, rnd, acc, names


def bound(ref, acc, out_bf16, names):
    rnd = UBF * (ref.abs() + acc) if out_bf16 else torch.zeros_like(ref)
    return Bound(ref, rnd, acc, names)


def _usage(got, ref, b):
    err = (got - ref).abs()
    u = (err - b.rnd).clamp_min(0) / b.acc.clamp_min(1e-300)
    return torch.where(torch.isnan(got) | torch.isnan(ref), torch.full_like(u, math.inf), u)


def check(case, what, got, b, alt=None, show=8):
    """Checks every element of `got` against Bound b; alt (NaN where there is none) is a second value an element may
    take instead (a dropped element, a ReLU mask decided within rounding of zero).  Returns the largest usage; raises
    AssertionError naming the case, the number of elements over the bound and the first coordinates."""
    got = got.detach().to("cpu", torch.float64)
    assert got.shape == b.ref.shape, (case, what, tuple(got.shape), tuple(b.ref.shape))
    u = _usage(got, b.ref, b)
    if alt is not None:
        ua = _usage(got, alt, b)
        u = torch.where(torch.isnan(alt), u, torch.minimum(u, ua))
    usage = u.max().item() if u.numel() else 0.0
    bad = (u > 1).nonzero()
    if bad.shape[0]:
        lines = []
        for ix in bad[:show].tolist():
            t = tuple(ix)
            coords = ", ".join(f"{n}={v}" for n, v in zip(b.names, t))
            lines.append(f"  ({coords}): got={got[t].item():.9g} ref={b.ref[t].item():.9g} "
                         f"bound={(b.rnd[t] + b.acc[t]).item():.3g} usage={u[t].item():.3g}")
        raise AssertionError(f"{case}: {what}: {bad.shape[0]} element(s) over the bound, bound usage {usage:.3g}\n"
                             + "\n".join(lines))
    return usage


def check_exact(case, what, got, ref, names, show=8):
    """Bit-exact comparison (values; -0 == +0)."""
    got = got.detach().to("cpu", torch.float64)
    ref = ref.to(torch.float64)
    assert got.shape == ref.shape, (case, what, tuple(got.shape), tuple(ref.shape))
    bad = (got != ref).nonzero()
    if bad.shape[0]:
        lines = [f"  ({', '.join(f'{n}={v}' for n, v in zip(names, ix))}): got={got[tuple(ix)].item():.9g} "
                 f"ref={ref[tuple(ix)].item():.9g}" for ix in bad[:show].tolist()]
        raise AssertionError(f"{case}: {what}: {bad.shape[0]} element(s) differ\n" + "\n".join(lines))


def f32(t):
    return t.float().double()


# ------------------------------------------------------------------------------------------------ grid mirrors
def rowmap_grid(M, C, sms, rows_per_thread=8):
    """(gx, gy) of the channel-group-stationary streaming kernels (mirror of seg_elementwise.cu's rowmap_grid)."""
    G = C // 8
    GB = min(G, 256)
    rows_par = 256 // GB
    gy = -(-G // GB)
    groups = -(-M // rows_par)
    gx = -(-groups // rows_per_thread)
    floor_blocks = -(-sms * 2 // gy)
    if gx < floor_blocks:
        gx = min(floor_blocks, groups)
    gx = max(1, min(gx, -(-sms * 8 // gy)))
    return gx, gy


def colreduce_grid(M, C, sms):
    """(gx, gy, cap) of bn_stats (mirror of colreduce_grid)."""
    G = C // 8
    GB = min(G, 256)
    rows_par = 256 // GB
    gy = -(-G // GB)
    cap = sms * 8 // gy + 1
    return max(1, min(-(-M // (rows_par * 4)), cap)), gy, cap


def reduce2_grid(M, C, sms):
    return rowmap_grid(M, C, sms, 32)


def fused_grid(M, C, sms, blocks_per_sm):
    gx, gy = rowmap_grid(M, C, sms, 16)
    return min(gx, max(1, sms * blocks_per_sm // gy)), gy


def rows_par(C):
    return 256 // min(C // 8, 256)


def fused_schedule(M, C, sms, blocks_per_sm):
    """Phase 1b of bn_bwd_fused_kernel: nb blocks per slab fold ncol = 2W columns, cpb columns per block."""
    nb, gy = fused_grid(M, C, sms, blocks_per_sm)
    W = min(C // 8, 256) * 8
    cpb = -(-2 * W // nb)
    return {"nb": nb, "slabs": gy, "W": W, "cpb": cpb, "idle_fold_blocks": max(0, nb - -(-2 * W // cpb))}


def bwd_chain_two_launch(M, C, sms):
    """bn_bwd_reduce: every thread sums its grid-strided rows, the block adds its row lanes, the fp64 atomics are exact,
    the total is rounded to fp32 once."""
    gx, _ = reduce2_grid(M, C, sms)
    return -(-M // (gx * rows_par(C))) + rows_par(C) + 1


def bwd_chain_fused(M, C, sms):
    """bn_bwd_fused: the occupancy (blocks per SM) is not visible from Python, so the thread chain is taken at one block
    per SM (the fewest blocks, the longest chain) and the fold of phase 1b over the block partials at eight (the most
    blocks), + the row lanes of the block fold and one spare."""
    gx_min, _ = fused_grid(M, C, sms, 1)
    gx_max, _ = fused_grid(M, C, sms, 8)
    return -(-M // (gx_min * rows_par(C))) + rows_par(C) + gx_max + 1


def fp32_keep(p):
    return float(torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(p, dtype=torch.float32)))


# ------------------------------------------------------------------------------------------------ BatchNorm forward
def exact_stats(x2d):
    """float64 (sum, sum of squares) of bf16-exact rows [M, C]: exact in float64 at the sizes of the sweep."""
    return torch.cat([x2d.sum(0), (x2d * x2d).sum(0)])


class BnStats:
    """Biased batch statistics from exact sums; eps is the kernel's fp32 value."""

    def __init__(self, stats, count, eps, clamp_eps):
        C = stats.numel() // 2
        self.mean = stats[:C] / count
        self.var = (stats[C:] / count - self.mean ** 2).clamp_min(0)
        e = float(torch.tensor(eps, dtype=torch.float32))
        self.istd = 1.0 / torch.sqrt(self.var.clamp_min(e) if clamp_eps else self.var + e)
        self.unbiased = self.var * count / (count - 1) if count > 1 else self.var
        self.count = count


def bn_train_ref(x2d, st, gamma, beta, res=None):
    """Pre-activation reference and allowance of bn_apply_train: gamma (x - mean) istd + beta (+ res) and
    K_APPLY u32 T.  ReLU is 1-Lipschitz, so the same allowance holds after it."""
    g, b = gamma.double(), beta.double()
    pre = g * (x2d - st.mean) * st.istd + b
    mag = g.abs() * st.istd * (x2d.abs() + st.mean.abs()) + b.abs()
    if res is not None:
        pre = pre + res
        mag = mag + res.abs()
    return pre, K_APPLY * U32 * mag


def bn_ss_ref(x2d, ss, res=None):
    """bn_apply with given fp32 scale/shift (exact inputs): x sc + sh (+ res), K_APPLY_SS u32 T."""
    C = x2d.shape[-1]
    sc, sh = ss[:C].double(), ss[C:].double()
    pre = x2d * sc + sh
    mag = (x2d * sc).abs() + sh.abs()
    if res is not None:
        pre = pre + res
        mag = mag + res.abs()
    return pre, K_APPLY_SS * U32 * mag


NAMES_MC = ("m", "c")


def apply_bound(pre, acc, relu):
    return bound(pre.clamp_min(0) if relu else pre, acc, True, NAMES_MC)


def check_apply(case, got, pre, acc, relu=True):
    return check(case, "bn apply", got.reshape(pre.shape), apply_bound(pre, acc, relu))


def check_dropout(case, got, pre, acc, p, units=None):
    """Dropout after ReLU.  The hash cannot be reproduced, so each element is either 0 where its reference is positive
    (dropped) or within the bound of ref / (1 - p) (kept; the keep scale adds KEEP_ROUNDINGS).  The dropped fraction
    among the elements whose reference is clearly positive must be within 5 sigma of p; `units` (same shape, one id
    per draw: (image, channel) for Dropout2d) makes the draws per unit, and a unit must be dropped entirely or not at
    all.  Returns (usage, dropped fraction, number of draws)."""
    got = got.detach().to("cpu", torch.float64).reshape(pre.shape)
    ref = pre.clamp_min(0)
    keep = fp32_keep(p)
    acc_k = keep * acc + KEEP_ROUNDINGS * U32 * keep * ref
    b = bound(ref * keep, acc_k, True, NAMES_MC)
    alt = torch.where(ref > 0, torch.zeros_like(ref), torch.full_like(ref, math.nan))
    usage = check(case, "dropout", got, b, alt=alt)
    clear = pre > (UBF * (pre.abs() + acc) + acc) * 2
    dropped = (got == 0) & clear
    if units is None:
        n, d = int(clear.sum()), int(dropped.sum())
    else:
        u = units.reshape(pre.shape)[clear]
        dr = dropped[clear].to(torch.int64)
        nu = int(units.max()) + 1
        tot = torch.zeros(nu, dtype=torch.int64).index_add_(0, u, torch.ones_like(dr))
        drp = torch.zeros(nu, dtype=torch.int64).index_add_(0, u, dr)
        mixed = ((drp > 0) & (drp < tot)).nonzero().flatten()
        if mixed.numel():
            raise AssertionError(f"{case}: dropout: {mixed.numel()} unit(s) partly dropped, e.g. unit {mixed[0].item()}")
        n, d = int((tot > 0).sum()), int((drp > 0).sum())
    assert n > 0, case
    frac = d / n
    sigma = math.sqrt(p * (1 - p) / n)
    if abs(frac - p) > 5 * sigma:
        raise AssertionError(f"{case}: dropout: dropped fraction {frac:.4f} over {n} draws, p = {p}, 5 sigma = {5 * sigma:.4f}")
    return usage, frac, n


def check_save(case, save, st):
    """save = (mean, istd) in fp32: K_COEF u32 relative."""
    ref = torch.cat([st.mean, st.istd])
    b = bound(ref, K_COEF * U32 * ref.abs(), False, ("i",))
    return check(case, "save (mean, istd)", save, b)


def check_scale_shift(case, ss, gamma, beta, mean, istd):
    """scale_shift = (gamma istd, beta - mean gamma istd): K_COEF u32 of |sc| and of |mean sc| + |beta|."""
    g, b = gamma.double(), beta.double()
    sc = g * istd
    ref = torch.cat([sc, b - mean * sc])
    mag = torch.cat([sc.abs(), (mean * sc).abs() + b.abs()])
    return check(case, "scale/shift", ss, bound(ref, K_COEF * U32 * mag, False, ("i",)))


def check_running(case, rm_new, rv_new, rm_old, rv_old, st, momentum):
    """(1 - m) r + m {mean, unbiased var} in float64 from the fp32 momentum; two roundings (the operands and the fp32
    result) of the terms' magnitudes."""
    m = float(torch.tensor(momentum, dtype=torch.float32))
    out = []
    for got, old, v in ((rm_new, rm_old, st.mean), (rv_new, rv_old, st.unbiased)):
        ref = (1 - m) * old.double() + m * v
        mag = ((1 - m) * old.double()).abs() + (m * v).abs()
        out.append(check(case, "running statistics", got, bound(ref, 2 * U32 * mag, False, ("c",))))
    return max(out)


# ------------------------------------------------------------------------------------------------ BatchNorm backward
def remask(x2d, gamma, beta, mean32, istd32):
    """The ReLU mask the out == NULL variants recompute: sign(x sc + sh) with the kernels' fp32 sc = gamma istd and
    sh = fma(-mean, sc, beta).  x sc is exact in float64, so the sign is exact up to sh, which is formed here by one
    float64 product-and-add rounded to fp32 (a double rounding the kernel's fma does not make): elements within 2 ulp(sh)
    of zero may take either mask value.  Returns (mask, ambiguous)."""
    sc = (gamma.float() * istd32.float()).double()
    sh = (-mean32.double() * sc + beta.double()).float()
    ulp = (torch.nextafter(sh.abs(), torch.tensor(math.inf)) - sh.abs()).double()
    v = x2d * sc + sh.double()
    return v > 0, v.abs() <= 2 * ulp


class BwdRef:
    """Reference of the BatchNorm backward.  dz' = dz [mask] keep; s0 = sum dz'; s1 = sum dz' xhat;
    dx = A (dz' - s0 / M - xhat s1 / M), A = gamma istd;  dres = beta_res old + dz'."""

    def __init__(self, dout, x2d, save, gamma, mask=None, keep=1.0, chain=1, ambiguous=None):
        C = x2d.shape[-1]
        M = x2d.shape[0]
        self.M = M
        mean, istd = save[:C].double(), save[C:].double()
        self.mean, self.istd = mean, istd
        m = torch.ones_like(dout) if mask is None else mask.double()
        self.dz = dout * m * keep
        xhat = (x2d - mean) * istd
        self.xhat, self.xabs = xhat, x2d.abs()
        t1 = self.dz * xhat
        self.s0, self.s1 = self.dz.sum(0), t1.sum(0)
        extra = KEEP_ROUNDINGS if keep != 1.0 else 0
        self.ds0 = (chain + extra) * U32 * self.dz.abs().sum(0)
        self.ds1 = (chain + 3 + extra) * U32 * t1.abs().sum(0)
        self.ambiguous = ambiguous
        if ambiguous is not None:  # a mask decided within rounding of zero may flip: its whole term
            a = ambiguous.double()
            self.ds0 = self.ds0 + (dout * keep * a).abs().sum(0)
            self.ds1 = self.ds1 + (dout * keep * a * xhat).abs().sum(0)
            self.dz_flip = torch.where(ambiguous, dout * keep * (1 - m), torch.full_like(dout, math.nan))
        self.A = gamma.double() * istd
        self.B = self.A * istd * self.s1 / M
        self.keep = keep

    def sums_bound(self):
        return bound(torch.cat([self.s0, self.s1]), torch.cat([self.ds0, self.ds1]), False, ("i",))

    def dx_bound(self, zero_sums=False):
        A, M = self.A, self.M
        if zero_sums:
            ref = A * self.dz
            acc = K_DX * U32 * (A * self.dz).abs()
        else:
            ref = A * (self.dz - self.s0 / M - self.xhat * self.s1 / M)
            acc = K_DX * U32 * ((A * self.dz).abs() + self.B.abs() * (self.xabs + self.mean.abs())
                                + (A * self.s0).abs() / M)
            acc = acc + A.abs() / M * (self.ds0 + self.xhat.abs() * self.ds1)
        return bound(ref, acc, True, NAMES_MC)

    def dx_alt(self, zero_sums=False):
        """dx with the ambiguous masks flipped (NaN elsewhere)."""
        if self.ambiguous is None:
            return None
        A, M = self.A, self.M
        d = self.dz_flip
        return A * d if zero_sums else A * (d - self.s0 / M - self.xhat * self.s1 / M)

    def dres_bound(self, beta_res=0.0, old=None):
        ref, mag = self.dz.clone(), self.dz.abs()
        if beta_res != 0.0:
            ref = ref + beta_res * old
            mag = mag + (beta_res * old).abs()
        return bound(ref, 3 * U32 * mag, True, NAMES_MC)

    def param_bound(self, which, old=None):
        """dbeta (which = 0) = s0 or dgamma (1) = s1, + old when accumulating (one more rounding)."""
        s, ds = (self.s0, self.ds0) if which == 0 else (self.s1, self.ds1)
        ref, acc = s.clone(), ds + U32 * s.abs()
        if old is not None:
            ref = ref + old.double()
            acc = acc + U32 * (s.abs() + old.double().abs())
        return bound(ref, acc, False, ("c",))


# ------------------------------------------------------------------------------------------------ max pool 3x3 s2 p1
NAMES_NHWC = ("n", "h", "w", "c")


def maxpool_ref(x):
    """x NHWC (bf16-exact) -> (y NHWC, tap NHWC int64: r * 3 + s of ATen's first maximum)."""
    N, H, W, C = x.shape
    y, ind = F.max_pool2d(nchw(x), 3, 2, 1, return_indices=True)
    P, Q = y.shape[2], y.shape[3]
    h, w = ind // W, ind % W
    p = torch.arange(P).view(1, 1, P, 1)
    q = torch.arange(Q).view(1, 1, 1, Q)
    tap = (h - (2 * p - 1)) * 3 + (w - (2 * q - 1))
    return nhwc(y), nhwc(tap)


def check_maxpool_fwd(case, y, idx, x):
    ry, rtap = maxpool_ref(x)
    check_exact(case, "maxpool y", y, ry, NAMES_NHWC)
    check_exact(case, "maxpool idx", idx.to(torch.int64), rtap, NAMES_NHWC)
    return 0.0


def maxpool_bwd_bound(dy, tap, x_shape):
    """dx = sum of dy over the windows whose (given) tap selects the pixel; each pixel is in at most 2 x 2 windows:
    3 u32 sum |dy| covers the fp32 adds."""
    N, H, W, C = x_shape
    P, Q = dy.shape[1], dy.shape[2]
    p = torch.arange(P).view(1, P, 1, 1)
    q = torch.arange(Q).view(1, 1, Q, 1)
    h = 2 * p - 1 + tap // 3
    w = 2 * q - 1 + tap % 3
    n = torch.arange(N).view(N, 1, 1, 1).expand_as(tap)
    c = torch.arange(C).view(1, 1, 1, C).expand_as(tap)
    flat = ((n * H + h) * W + w) * C + c
    ref = torch.zeros(N * H * W * C, dtype=torch.float64).index_add_(0, flat.flatten(), dy.double().flatten())
    mag = torch.zeros(N * H * W * C, dtype=torch.float64).index_add_(0, flat.flatten(), dy.double().abs().flatten())
    return bound(ref.view(x_shape), 3 * U32 * mag.view(x_shape), True, NAMES_NHWC)


# ------------------------------------------------------------------------------------------------ adaptive avg pool
def bin_edges(L, b):
    """ATen's adaptive pooling bins: [floor(i L / b), ceil((i + 1) L / b))."""
    return [((i * L) // b, -(-(i + 1) * L // b)) for i in range(b)]


def avgpool_fwd_bound(x, bins):
    """Forward: (ceil(cnt / 8) + 8 + 2) u32 sum|x| / cnt: 8 pixel lanes each sum ceil(cnt / 8) pixels, the shared
    memory fold adds the 8 lanes, then one division (+ 1 spare)."""
    N, H, W, C = x.shape
    ref = nhwc(F.adaptive_avg_pool2d(nchw(x), bins))
    mag = nhwc(F.adaptive_avg_pool2d(nchw(x.abs()), bins))
    k = torch.zeros(1, bins, bins, 1, dtype=torch.float64)
    for i, (h0, h1) in enumerate(bin_edges(H, bins)):
        for j, (w0, w1) in enumerate(bin_edges(W, bins)):
            k[0, i, j, 0] = -(-(h1 - h0) * (w1 - w0) // 8) + 8 + 2
    return bound(ref, k * U32 * mag, True, NAMES_NHWC)


def avgpool_bwd_bound(dy, x_shape, bins, beta=0.0, old=None):
    """Backward: sum over the <= 2 x 2 bins containing the pixel of dy fp32(1 / cnt) (+ beta old):
    (taps + 2) u32 of the terms' magnitudes."""
    N, H, W, C = x_shape
    dyd = dy.double()
    ref = torch.zeros(x_shape, dtype=torch.float64)
    mag = torch.zeros(x_shape, dtype=torch.float64)
    taps = torch.zeros(1, H, W, 1, dtype=torch.float64)
    for i, (h0, h1) in enumerate(bin_edges(H, bins)):
        for j, (w0, w1) in enumerate(bin_edges(W, bins)):
            cnt = (h1 - h0) * (w1 - w0)
            ref[:, h0:h1, w0:w1] += dyd[:, i:i + 1, j:j + 1] / cnt
            mag[:, h0:h1, w0:w1] += dyd[:, i:i + 1, j:j + 1].abs() / cnt
            taps[:, h0:h1, w0:w1] += 1
    acc = (taps + 2) * U32 * mag
    if beta != 0.0:
        ref = ref + beta * old
        acc = acc + 2 * U32 * (beta * old).abs()
    return bound(ref, acc, True, NAMES_NHWC)


# ------------------------------------------------------------------------------------------------ bilinear
def lerp_axis(inp, out, align_corners):
    """(i0, i1, l1, l0) per output index exactly as ATen's area_pixel_compute_source_index for float tensors and as
    the kernel: float32 scale, float32 source index, clamps.  The source index scale (dst + 0.5) - 0.5 is one fused
    multiply-add in both (nvcc contracts it, and so do ATen's vectorised CPU kernels): it is formed here as the exact
    float64 product-and-add rounded once to float32."""
    f = torch.float32
    d = torch.arange(out, dtype=f)
    if align_corners:
        scale = (torch.tensor(float(inp - 1), dtype=f) / torch.tensor(float(out - 1), dtype=f)) if out > 1 \
            else torch.tensor(0.0, dtype=f)
        s = scale * d
    else:
        scale = torch.tensor(float(inp), dtype=f) / torch.tensor(float(out), dtype=f)
        s = (scale.double() * (d + 0.5).double() - 0.5).to(f).clamp_min(0)
    i0 = s.to(torch.int64).clamp_max(inp - 1)
    i1 = torch.where(i0 < inp - 1, i0 + 1, i0)
    l1 = s - i0.to(f)
    l0 = 1 - l1
    return i0, i1, l1, l0


def lerp_matrix(inp, out, align_corners):
    """[out, inp] float64 interpolation matrix of one axis (weights are the fp32 lambdas)."""
    i0, i1, l1, l0 = lerp_axis(inp, out, align_corners)
    A = torch.zeros(out, inp, dtype=torch.float64)
    r = torch.arange(out)
    A.index_put_((r, i0), l0.double(), accumulate=True)
    A.index_put_((r, i1), l1.double(), accumulate=True)
    return A


def outputs_per_input(inp, out, align_corners):
    """Largest number of consecutive outputs an input index feeds (first to last output with a non-zero fp32 weight,
    as bilinear_bwd_kernel's lerp_weights counts them); more than MAXN takes the kernel's fallback loop."""
    i0, i1, l1, l0 = lerp_axis(inp, out, align_corners)
    n = 0
    for y in range(inp):
        wy = torch.where(i0 == y, l0, torch.zeros_like(l0)) + torch.where(i1 == y, l1, torch.zeros_like(l1))
        nz = (wy != 0).nonzero().flatten()
        if nz.numel():
            n = max(n, int(nz[-1] - nz[0]) + 1)
    return n


def bilinear_fwd_bound(x, Ho, Wo, align_corners, out_bf16=True):
    """x NHWC -> NHWC; 6 u32 sum |w x| (two lerps of two fp32 products and adds each) + the output rounding."""
    N, Hi, Wi, C = x.shape
    Ay, Ax = lerp_matrix(Hi, Ho, align_corners), lerp_matrix(Wi, Wo, align_corners)
    ref = torch.einsum("oh,nhwc,pw->nopc", Ay, x.double(), Ax)
    mag = torch.einsum("oh,nhwc,pw->nopc", Ay.abs(), x.double().abs(), Ax.abs())
    return bound(ref, 6 * U32 * mag, out_bf16, NAMES_NHWC)


def bilinear_bwd_bound(dy, Hi, Wi, align_corners, beta=0.0, old=None):
    """dy NHWC [N, Ho, Wo, C] -> dx NHWC [N, Hi, Wi, C] = Ay^T dy Ax (+ beta old): (taps + 2) u32 sum |w dy|, taps =
    the number of (oy, ox) pairs that reference the input pixel."""
    N, Ho, Wo, C = dy.shape
    Ay, Ax = lerp_matrix(Hi, Ho, align_corners), lerp_matrix(Wi, Wo, align_corners)
    ref = torch.einsum("oh,nopc,pw->nhwc", Ay, dy.double(), Ax)
    mag = torch.einsum("oh,nopc,pw->nhwc", Ay.abs(), dy.double().abs(), Ax.abs())
    taps = ((Ay != 0).sum(0).view(Hi, 1) * (Ax != 0).sum(0).view(1, Wi)).double().view(1, Hi, Wi, 1)
    acc = (taps + 2) * U32 * mag
    if beta != 0.0:
        ref = ref + beta * old
        acc = acc + 2 * U32 * (beta * old).abs()
    return bound(ref, acc, True, NAMES_NHWC)


# ------------------------------------------------------------------------------------------------ ReLU, axpby
def relu_fwd_ref(x):
    return x.clamp_min(0)


def relu_bwd_bound(dy, y, beta=0.0, old=None):
    """dx = dy [y > 0] (+ beta old): exact up to the fp32 beta old + v and its bf16 rounding."""
    d = torch.where(y > 0, dy.double(), torch.zeros_like(dy.double()))
    return axpby_bound(d, beta, old)


def axpby_bound(v, beta=0.0, old=None):
    """y = v + beta old: two fp32 roundings of the terms, then bf16."""
    ref, mag = v.double().clone(), v.double().abs()
    if beta != 0.0:
        ref = ref + beta * old
        mag = mag + (beta * old).abs()
    return bound(ref, 2 * U32 * mag, True, ("m", "c") if v.dim() == 2 else NAMES_NHWC)
