"""Per-element conformance checker for the convolution kernels (fprop, dgrad, wgrad).

Pure torch on the CPU; it imports nothing from the library, so its own tests run without a GPU
(test_conv_check_cpu.py) and the GPU sweep (test_conv_conformance_gpu.py) feeds it what the kernels wrote.

Reference: the float64 convolution of the bf16-rounded operands.  Magnitude A: the same operation on |operands|.
Per-element bound (u32 = 2^-24, u_bf16 = 2^-8; n = the contraction length, A = the magnitude):

    |got - ref| <= r + e,   e = u32 |ref| + kappa(n) u32 (A + |bias| + |beta old|)          (accumulation allowance)
                            r = 0 (fp32 outputs);  u_bf16 |ref|  (bf16 outputs)             (rounding allowance)
                                + u_bf16 |conv + bias|  (bf16 outputs with beta != 0 on the wgmma path, whose epilogue
                                                  rounds the convolution (+ bias) to bf16 before it adds beta * old)

"Bound usage" of an element is (|got - ref| - r)+ / e: the share of the accumulation allowance the element needs after
its allowed roundings.  An element fails when its usage exceeds 1; a case reports its largest usage.

Statistics (BatchNorm sums the conv epilogue produces) are checked per channel and per half against the float64 sums
of the values read back from the output as stored: |S[c] - sum| <= chain u32 sum|.|, chain = the length of the longest
fp32 summation chain of the kernel (see stat_chain_tc / stat_chain_simt).
"""
import math

import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

U32 = 2.0 ** -24
UBF = 2.0 ** -8
BM = 128       # output rows per tile of the wgmma kernels
GUARD = 8      # guard channels on each side of a guarded slice
# The longest fp32 contractions of the GPU sweep (which asserts it stays within them): the checker's self-tests show that
# one dropped product is still caught at these lengths, where the bound is widest.
LARGEST_FPROP_F32_N = 9 * 304
LARGEST_WGRAD_PIXELS = 132 * 132


def kappa(n, splits=0):
    """Roundings charged to the accumulation of an n-long dot product.

    The wgmma kernels multiply bf16 operands (the products are exact in fp32) and add them into fp32 accumulators one
    k16 MMA step at a time: ceil(n / 16) steps, each modelled as one fp32 rounding of a partial sum whose magnitude is
    at most A, hence ceil(n / 16) * u32 * A.  The + 16 is slack for what that model leaves out: the tensor core's
    alignment of the 16 products inside a step (a few extra roundings relative to A), the bias and beta additions
    (one rounding each) and the different summation orders of the CUDA-core kernel and of ATen's CPU convolution
    (which charge more roundings in the worst case, but whose errors on random-sign data grow like sqrt(n), far below
    this).  wgrad's split-K adds one fp32 addition per split in the reduction, hence + splits.
    Changing this constant needs a written reason, and test_conv_check_cpu.py's sensitivity tests must still pass."""
    return math.ceil(n / 16) + 16 + splits


def stat_rows_for(ncols):
    """Rows per fp32 group of the wgmma epilogue's statistics fold (mirror of seg_conv_tc.cu's stat_rows_for)."""
    if ncols <= 64:
        return 32
    if ncols < 256:
        return 64
    return 128 if math.ceil(ncols / 256) * 256 - ncols < 128 else 64


def stat_chain_tc(ncols):
    """Longest fp32 summation chain of the wgmma statistics: stat_rows rows per group, then the 128 / stat_rows group
    sums of a tile, then one rounding to spare (the tiles' fp32 partials are added exactly in fp64)."""
    sr = stat_rows_for(ncols)
    return sr + BM // sr + 1


def stat_chain_simt(M, ncols, sms):
    """Longest fp32 summation chain of bn_stats (the CUDA-core path's statistics): every thread sums its grid-strided
    rows, then a block adds its row lanes (mirror of seg_elementwise.cu's colreduce_grid)."""
    G = ncols // 8
    GB = min(G, 256)
    rows_par = 256 // GB
    gy = -(-G // GB)
    gx = max(1, min(-(-M // (rows_par * 4)), sms * 8 // gy + 1))
    return -(-M // (gx * rows_par)) + rows_par + 1


# ------------------------------------------------------------------------------------------------ operands
def bf16_round(t):
    return t.to(torch.bfloat16).to(torch.float64)


def channel_scales(n, seed):
    """Per-channel magnitudes 2^0 .. 2^-9 so that every case has low-magnitude channels next to large ones (an error
    there is invisible to a max-normalised check)."""
    g = torch.Generator().manual_seed(seed)
    return 2.0 ** -(3 * torch.randint(0, 4, (n,), generator=g)).to(torch.float64)


def make_x(N, H, W, C, seed):
    """NHWC activations (bf16-exact float64) with per-channel magnitudes."""
    g = torch.Generator().manual_seed(seed)
    return bf16_round(torch.randn(N, H, W, C, generator=g, dtype=torch.float64) * channel_scales(C, seed + 1))


def make_w(K, C, R, S, seed):
    """OIHW weights (bf16-exact float64), fan-in normalised, with per-output-channel magnitudes."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(K, C, R, S, generator=g, dtype=torch.float64) / math.sqrt(C * R * S)
    return bf16_round(w * channel_scales(K, seed + 1).view(K, 1, 1, 1))


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def pack_w(w_oihw):
    """OIHW -> packed [R*S][K][C] (the layout of the library's weights and weight gradients)."""
    K, C, R, S = w_oihw.shape
    return w_oihw.permute(2, 3, 0, 1).reshape(R * S, K, C)


# ------------------------------------------------------------------------------------------------ references
class Ref:
    """ref: exact result; staged: the convolution (+ bias) before beta old is added; mag: A; extra: |bias| + |beta old|;
    n: contraction length."""

    def __init__(self, ref, staged, mag, extra, n, coord_names):
        self.ref, self.staged, self.mag, self.extra, self.n, self.coord_names = ref, staged, mag, extra, n, coord_names


def fprop_ref(x, w, stride, pad, dil, bias=None, beta=0.0, old=None):
    """x: NHWC, w: OIHW (bf16-exact values); returns NHWC float64 [N, P, Q, K]."""
    xd, wd = nchw(x.double()), w.double()
    conv = nhwc(F.conv2d(xd, wd, None, stride, pad, dil))
    mag = nhwc(F.conv2d(xd.abs(), wd.abs(), None, stride, pad, dil))
    ref, extra = conv.clone(), torch.zeros_like(conv)
    if bias is not None:
        ref += bias.double()
        extra += bias.double().abs()
    staged = ref.clone()
    if beta != 0.0:
        ref += beta * old.double()
        extra += (beta * old.double()).abs()
    K, C, R, S = w.shape
    return Ref(ref, staged, mag, extra, R * S * C, ("n", "h", "w", "c"))


def dgrad_ref(dy, w, x_shape, stride, pad, dil, beta=0.0, old=None):
    """dy: NHWC [N, P, Q, K], w: OIHW; returns NHWC float64 [N, H, W, C] = beta old + conv_transpose(dy, w)."""
    N, H, W, C = x_shape
    dyd, wd = nchw(dy.double()), w.double()
    size = (N, C, H, W)
    conv = nhwc(nn_grad.conv2d_input(size, wd, dyd, stride, pad, dil))
    mag = nhwc(nn_grad.conv2d_input(size, wd.abs(), dyd.abs(), stride, pad, dil))
    ref, extra = conv.clone(), torch.zeros_like(conv)
    if beta != 0.0:
        ref += beta * old.double()
        extra += (beta * old.double()).abs()
    K, _, R, S = w.shape
    return Ref(ref, conv, mag, extra, R * S * K, ("n", "h", "w", "c"))


def wgrad_ref(dy, x, R, S, stride, pad, dil, old=None):
    """dy: NHWC [N, P, Q, K], x: NHWC [N, H, W, C]; returns packed float64 [R*S][K][C] = old + dy^T im2col(x)."""
    K, C = dy.shape[-1], x.shape[-1]
    dyd, xd = nchw(dy.double()), nchw(x.double())
    conv = pack_w(nn_grad.conv2d_weight(xd, (K, C, R, S), dyd, stride, pad, dil))
    mag = pack_w(nn_grad.conv2d_weight(xd.abs(), (K, C, R, S), dyd.abs(), stride, pad, dil))
    ref, extra = conv.clone(), torch.zeros_like(conv)
    if old is not None:
        ref += old.double()
        extra += old.double().abs()
    return Ref(ref, conv, mag, extra, dy.shape[0] * dy.shape[1] * dy.shape[2], ("tap", "k", "c"))


# ------------------------------------------------------------------------------------------------ bounds
def allowances(r, out_bf16, staged=False, splits=0):
    """(rounding allowance, accumulation allowance) per element of Ref r."""
    aref = r.ref.abs()
    acc = U32 * aref + kappa(r.n, splits) * U32 * (r.mag + r.extra)
    rnd = torch.zeros_like(aref)
    if out_bf16:
        rnd = rnd + UBF * aref
        if staged:
            rnd = rnd + UBF * r.staged.abs()
    return rnd, acc


def _fail(case, what, idx, lines, nbad, usage):
    raise AssertionError(f"{case}: {what}: {nbad} element(s) over the bound, bound usage {usage:.3g}\n" + "\n".join(lines))


def check_elements(case, got, r, out_bf16, staged=False, splits=0, show=8):
    """Checks every element of `got` (any float tensor of r.ref's shape) against the bound; returns the case's
    largest bound usage.  Raises AssertionError naming the case, the number of elements over the bound, the first
    few coordinates with got / ref / bound, and the largest usage."""
    got = got.detach().to("cpu", torch.float64)
    assert got.shape == r.ref.shape, (case, tuple(got.shape), tuple(r.ref.shape))
    rnd, acc = allowances(r, out_bf16, staged, splits)
    err = (got - r.ref).abs()
    usage_t = (err - rnd).clamp_min(0) / acc.clamp_min(1e-300)
    usage_t = torch.where(torch.isnan(got), torch.full_like(usage_t, math.inf), usage_t)
    usage = usage_t.max().item() if usage_t.numel() else 0.0
    bad = (usage_t > 1).nonzero()
    if bad.shape[0]:
        lines = []
        for ix in bad[:show].tolist():
            t = tuple(ix)
            coords = ", ".join(f"{n}={v}" for n, v in zip(r.coord_names, t))
            lines.append(f"  ({coords}): got={got[t].item():.9g} ref={r.ref[t].item():.9g} "
                         f"bound={(rnd[t] + acc[t]).item():.3g} usage={usage_t[t].item():.3g}")
        _fail(case, "elements", bad, lines, bad.shape[0], usage)
    return usage


def check_stats(case, stats, stored, chain, show=8):
    """stats: the kernel's fp64 [2K] (sum, sum of squares); stored: [M, K] values read back from the output.  Checks
    each channel and half on its own; returns the largest bound usage."""
    s = stats.detach().to("cpu", torch.float64)
    y = stored.detach().to("cpu", torch.float64).reshape(-1, stored.shape[-1])
    K = y.shape[1]
    exact = torch.cat([y.sum(0), (y * y).sum(0)])
    mag = torch.cat([y.abs().sum(0), (y * y).sum(0)])
    bound = chain * U32 * mag
    err = (s - exact).abs()
    usage_t = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    usage_t = torch.where(torch.isnan(s), torch.full_like(usage_t, math.inf), usage_t)
    usage = usage_t.max().item()
    bad = (usage_t > 1).nonzero().flatten()
    if bad.numel():
        lines = [f"  ({'sum' if i < K else 'sum of squares'}, c={i % K}): got={s[i].item():.12g} "
                 f"exact={exact[i].item():.12g} bound={bound[i].item():.3g}" for i in bad[:show].tolist()]
        _fail(case, "statistics", bad, lines, bad.numel(), usage)
    return usage


# ------------------------------------------------------------------------------------------------ guarded buffers
SENTINEL_BITS = {torch.bfloat16: 0x7FA5, torch.float32: 0x7FA5A5A5,  # NaN bit patterns (quiet bit clear: no kernel makes them)
                 torch.int64: 0x5A5A5A5A5A5A5A5A}  # int64 label maps: outside the int32 range every label comes from
_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}


def sentinel_fill(t):
    """Fill a bf16 / fp32 tensor with the sentinel bit pattern."""
    t.view(_INT[t.dtype]).fill_(SENTINEL_BITS[t.dtype])
    return t


def is_sentinel(t):
    return t.view(_INT[t.dtype]) == SENTINEL_BITS[t.dtype]


class Guarded:
    """An NHWC tensor [N, H, W, C] living at channel offset `lead` of a buffer [N + 1, H, W, lead + C + trail]: `lead`
    and `trail` guard channels on each side of every pixel (0 for a dense tensor) and one trailing guard image.  The
    whole buffer starts as the sentinel; `view` is what the kernel gets."""

    def __init__(self, N, H, W, C, dtype, lead=GUARD, trail=GUARD, device="cpu"):
        self.N, self.lead, self.C = N, lead, C
        self.buf = sentinel_fill(torch.empty(N + 1, H, W, lead + C + trail, dtype=dtype, device=device))
        self.view = self.buf[:N, :, :, lead:lead + C]

    def guard_mask(self):
        m = torch.ones(self.buf.shape, dtype=torch.bool)
        m[:self.N, :, :, self.lead:self.lead + self.C] = False
        return m


class FlatGuarded:
    """A dense tensor of `shape` at element offset `lead` of a flat buffer with `lead` / `trail` sentinel words around
    it (the weight gradient [R*S][K][C] has no pitch to put guards in)."""

    def __init__(self, shape, dtype, lead=GUARD, trail=GUARD, device="cpu"):
        n = math.prod(shape)
        self.lead, self.n = lead, n
        self.buf = sentinel_fill(torch.empty(lead + n + trail, dtype=dtype, device=device))
        self.view = self.buf[lead:lead + n].view(shape)

    def guard_mask(self):
        m = torch.ones(self.buf.shape, dtype=torch.bool)
        m[self.lead:self.lead + self.n] = False
        return m


def check_guards(case, buf, guard_mask, show=8):
    """Every guard word of `buf` must still hold the sentinel, bit for bit."""
    b = buf.detach().cpu()
    changed = (~is_sentinel(b)) & guard_mask
    n = int(changed.sum())
    if n:
        lines = [f"  guard word {tuple(ix)} = {b[tuple(ix)].item()!r}" for ix in changed.nonzero()[:show].tolist()]
        raise AssertionError(f"{case}: {n} guard word(s) overwritten\n" + "\n".join(lines))


def check_written(case, view, show=8):
    """No element of the logical region may still hold the sentinel (it was never written)."""
    v = view.detach().cpu()
    left = is_sentinel(v)
    n = int(left.sum())
    if n:
        lines = [f"  (n, h, w, c)={tuple(ix)} still holds the sentinel" for ix in left.nonzero()[:show].tolist()]
        raise AssertionError(f"{case}: {n} element(s) never written\n" + "\n".join(lines))
