"""Per-element conformance checker for the loss and metric kernels of seg_loss.cu and seg_lovasz.cu on NCHW fp32 logits:
cross-entropy, class-weighted CE and focal loss (forward sums and logits gradient), Dice (forward and gradient),
Lovász-softmax (loss and gradient, and the order of tied errors) and eval_metrics (arg-max and counters).

Pure torch, like conv_check.py and elementwise_check.py, whose guarded buffers, sentinels and element checks it reuses:
its own tests run without a GPU (test_loss_check_cpu.py) and the GPU sweep (test_loss_conformance_gpu.py) feeds it what
the kernels wrote.  Every reference is float64 of the fp32 logits and runs on the device the logits are on (the sweep
computes its large references on the GPU, in float64).

Per-element bound (u32 = 2^-24):  |got - ref| <= e, with e counted from the kernel's fp32 roundings.

Softmax of one pixel (every kernel forms it the same way: mx = max_c z_c, se = sum_c expf(z_c - mx) serially,
inv = 1 / se, p_c = expf(z_c - mx) * inv; CUDA's expf is within 2 ulp = 4 u32 relative, the build has no fast math):
    z_c - mx rounds once, which perturbs expf's result by u32 |z_c - mx| relative;
    se:  rel_se = (C - 1 adds + 4 expf + sum_c p_c |z_c - mx|) u32,
    p_c: rel_p  = rel_se + (4 expf + |z_c - mx| + inv + product) u32, charged as (C + 12 + 3 |z_c - mx| + w_se) u32:
         ATen's float32 path forms p as exp(z_c - mx - log se) and rounds a quantity of size |z_c - mx| three times,
         and the checker must accept it as a correct result.
nll = (mx + logf(se)) - z_t:  e_nll = rel_se + 3 u32 (|mx| + |log se| + |z_t|)  (logf is within 1 ulp; the two
    additions round once each).
CE / weighted CE gradient (p_c - [c = t]) g w_t:  |g w_t| (rel_p p_c + u32 |p_c - [c = t]|) + 3 u32 |ref|  (g = gs / D,
    gp = g w_t and the final product round once each; p_t - 1 cancels, so the allowance scales with p_c).
Focal F(L) = u^gamma L and F'(L) = u^gamma (1 + gamma r), u = -expm1(-L), r = L / expm1(L), L = w_t nll:
    L carries e_L = w_t e_nll + u32 L.  F and F' are evaluated in float64 at L - e_L, L and L + e_L and the spread is
    charged (a derivative bound fails: for gamma < 1, F'' is unbounded at L -> 0), plus their own roundings relative to
    the value: K_F = 10 + 4 gamma (expm1f 1 ulp raised to gamma, powf 4 ulp, the product) and K_FP = 16 + 4 gamma
    (r: expm1f and a division; 1 + gamma r: two; powf; two products).
Reductions: the loss and the denominator are fp64 sums of fp32 per-pixel terms; the fp32 terms are charged (their
    allowances add up), the fp64 sum gets n 2^-53 sum |term|.  The denominators are exact integers (CE: valid pixels;
    focal: all pixels) or sums of fp32 weights (weighted CE), which fp64 adds exactly at these sizes: checked exactly.
Dice: D = 2 npix + smooth in the kernel; the reference's sum(softmax) + npix + smooth equals it to within the p
    allowance.  I = sum_pixels p_t gets sum rel_p p_t; the gradient -(2 / D) gs p_t ([c = t] - p_c) gets the p
    allowances of both factors and 4 roundings.
Lovász (per present class c, over the valid pixels in flat pixel order): errors e_i = |fg_i - p_ic| with allowance
    delta_i = rel_p p_ic + u32 e_i (1 - p rounds for foreground).  The kernel's order comes from its fp32 errors, so
    the check tolerates every order fp32 rounding can produce: sort the float64 errors stably (descending; pixel order
    among ties); split the sorted list into clusters at every point where all intervals [e - delta, e + delta] before it
    lie strictly above all intervals after it.  Inside a cluster any order is legitimate.  With G foreground pixels in
    the class and F0 / B0 foreground / background pixels ranked before a cluster holding nf / nb of each, a member's
    d = J_i - J_{i-1} (J = (cf + cb) / (G + cb) after cf foreground and cb background ranks) lies in
        foreground: [1 / (G + B0 + nb),  1 / (G + B0)]
        background: [(G - F0 - nf) / ((G + B0 + nb - 1)(G + B0 + nb)),  (G - F0) / ((G + B0)(G + B0 + 1))]
    (the foreground step 1 / (G + cb) depends only on the background before it; the background step
    (G - cf) / ((G + cb)(G + cb + 1)) falls as either count grows).  d itself is a difference of two fp32 Jaccard values
    near 1, each formed with a division and a subtraction: 5 u32 absolute.  The gradient p_c (g_c - sum_k p_k g_k) /
    n_present, g = -d (foreground) or +d (background), gets the interval's radius and d's rounding propagated through it,
    the p allowances, and C + 4 roundings of the dot product and products.
    The loss is 1-Lipschitz in the max-norm of the errors (d >= 0, sum d <= 1), so a class's loss is within
    max delta_i + 4 u32 of the float64 value whatever the order (the d roundings telescope to 2 u32 max e; 2 more for the
    products); the mean gets one more rounding.
    Where an error lies within its allowance of 0, |fg - p| has no derivative: the kernel takes -1 / +1, ATen's abs
    backward 0; the member's g may be either.
    Tie order (the contract of seg_lovasz.cu): exactly tied errors take ranks in flat pixel order.  With
    tie_order=True a cluster whose members all have the same float64 error (bit-identical logits, or saturated
    probabilities) is held to that order: each member's d is the one of its stable rank.
Metrics: the arg-max is the first maximum; the counters are exact.

Schedule mirrors (nchw_grid, lovasz_schedule) copy the host grid functions of seg_loss.cu and seg_lovasz.cu so that
the sweep can assert the regime each case names.
"""
import math

import torch
import torch.nn.functional as F

from conv_check import U32, FlatGuarded, check_guards, check_written, sentinel_fill  # noqa: F401
from conv_check import UBF
from elementwise_check import Bound, bound, check, check_exact, lerp_axis, lerp_matrix  # noqa: F401

NAMES = ("n", "c", "h", "w")
K_P = 12  # softmax p_c: C + K_P + 3 |z_c - mx| + w_se roundings (derivation in the module docstring)
D_ROUND = 5  # Lovász d = J_i - J_{i-1}: absolute allowance in u32
# fp32 underflow: expf results and products below 2^-126 lose relative precision (subnormals, flush to 0); every p_c
# gets this absolute allowance on top of the relative one, and every fp32 output the absolute SUB.
TINY = 2.0 ** -125
SUB = 2.0 ** -148
LV_MAXC, LV_TILE, LV_JT = 256, 256 * 32, 4096
FUSED_MAXC = 160
# An int32 / int64 word no kernel writes: outputs that must be written are pre-filled with it.
INT_SENTINEL = {torch.int32: -0x5A5A5A5B, torch.int64: -0x5A5A5A5A5A5A5A5B}


def int_sentinel_fill(t):
    return t.fill_(INT_SENTINEL[t.dtype])


def check_int_guards(case, buf, lead, n, show=8):
    """Every word of the int buffer outside [lead, lead + n) must still hold the int sentinel."""
    b = buf.detach().cpu()
    m = torch.ones(b.shape, dtype=torch.bool)
    m[lead:lead + n] = False
    bad = ((b != INT_SENTINEL[b.dtype]) & m).nonzero().flatten()
    if bad.numel():
        raise AssertionError(f"{case}: {bad.numel()} guard word(s) overwritten: "
                             + ", ".join(f"[{i}]={b[i].item()}" for i in bad[:show].tolist()))


# ------------------------------------------------------------------------------------------------ schedule mirrors
def nchw_grid(npix, sms):
    """Blocks of ce_nchw_*, dice_nchw_*, eval_metrics (and the shuffle loss): min(ceil(npix / 256), 8 SMs); returns
    (blocks, grid-stride iterations of the busiest thread, capped)."""
    want = max(1, -(-npix // 256))
    blocks = min(want, sms * 8)
    return blocks, -(-npix // (blocks * 256)), want > sms * 8


def lovasz_schedule(npix, P, n_present, sms):
    """Grids of seg_lovasz.cu for npix pixels, P valid, n_present present classes."""
    nkeys = P * n_present
    nblocks = -(-nkeys // LV_TILE)
    tiles = -(-P // LV_JT)
    nchunks = -(-npix // 256)
    return {"count_blocks": max(1, min(-(-npix // 2048), sms * 4)),
            "emit_blocks": min(nchunks, sms * 8), "chunks": nchunks, "emit_iters": -(-nchunks // min(nchunks, sms * 8)),
            "chunk_scan_per": -(-nchunks // 1024),
            "nblocks": nblocks, "radix_per": -(-nblocks // 1024), "tiles": tiles, "class_scan_per": -(-tiles // 1024)}


# ------------------------------------------------------------------------------------------------ softmax
class Softmax:
    """float64 softmax of NCHW logits z with the kernels' allowances (absolute, per element).  ev: None when z is what
    the kernel reads (fp32 or bf16 values), else the absolute allowance of the logits the kernel computed itself (the
    fused upsample's interpolation); a perturbation dv of the logits moves p_c by p_c (|dv_c| + sum_k p_k |dv_k|) and nll
    by |dv_t| + sum_k p_k |dv_k| to first order."""

    def __init__(self, z, ev=None):
        z = z.double()
        C = z.shape[1]
        self.z = z
        self.mx = z.amax(1, keepdim=True)
        self.dd = (z - self.mx).abs()
        ex = torch.exp(z - self.mx)
        self.se = ex.sum(1, keepdim=True)
        self.p = ex / self.se
        w_se = (self.dd * self.p).sum(1, keepdim=True)
        self.rel_se = (C + 4 + w_se) * U32
        self.ep = (C + K_P + 3 * self.dd + w_se) * U32 * self.p + TINY
        self.lse = self.mx + torch.log(self.se)
        self.ev, self.sev = ev, None
        if ev is not None:
            self.sev = (self.p * ev).sum(1, keepdim=True)
            self.ep = self.ep + self.p * (ev + self.sev)


def first_argmax(z):
    """Index of the first maximum along dim 1."""
    C = z.shape[1]
    idx = torch.arange(C, device=z.device).view(1, C, *([1] * (z.dim() - 2)))
    return torch.where(z == z.amax(1, keepdim=True), idx, C).amin(1)


def _safe_t(target, ignore, C):
    valid = target != ignore
    return valid, torch.where(valid, target, torch.zeros_like(target)).clamp(0, C - 1)


def nll_parts(sm, target, ignore):
    C = sm.z.shape[1]
    valid, t = _safe_t(target, ignore, C)
    zt = sm.z.gather(1, t.unsqueeze(1)).squeeze(1)
    lse = sm.lse.squeeze(1)
    nll = lse - zt
    e_nll = sm.rel_se.squeeze(1) + 3 * U32 * (sm.mx.squeeze(1).abs() + torch.log(sm.se.squeeze(1)).abs() + zt.abs())
    if sm.ev is not None:
        e_nll = e_nll + sm.ev.gather(1, t.unsqueeze(1)).squeeze(1) + sm.sev.squeeze(1)
    return valid, t, nll, e_nll


# ------------------------------------------------------------------------------------------------ CE / WCE / focal
def focal_F(L, gamma):
    return (-torch.expm1(-L)) ** gamma * L


def focal_Fp(L, gamma):
    u = -torch.expm1(-L)
    r = torch.where(L > 0, L / torch.expm1(L.clamp_min(1e-300)), torch.ones_like(L))
    return u ** gamma * (1 + gamma * r)


def _spread(f, L, eL, gamma):
    lo, mid, hi = f((L - eL).clamp_min(0), gamma), f(L, gamma), f(L + eL, gamma)
    return mid, torch.maximum((lo - mid).abs(), (hi - mid).abs()), torch.maximum(torch.maximum(lo, mid), hi)


class LossRef:
    """Per-pixel loss references of kind 'ce', 'wce' or 'focal' (weight: float [C] or None; gamma for focal)."""

    def __init__(self, z, target, ignore, kind, weight=None, gamma=0.0, mean=True, ev=None):
        self.sm = sm = Softmax(z, ev)
        C = sm.z.shape[1]
        dev = sm.z.device
        valid, t, nll, e_nll = nll_parts(sm, target, ignore)
        w = torch.ones(C, dtype=torch.float64, device=dev) if weight is None else weight.to(dev).double()
        wt = w[t] * valid if kind != "ce" else valid.double()
        self.valid, self.t, self.kind, self.mean = valid, t, kind, mean
        if kind == "focal":
            L = wt * nll
            eL = wt * e_nll + U32 * L
            F, dF, Fhi = _spread(focal_F, L, eL, gamma)
            Fp, dFp, Fphi = _spread(focal_Fp, L, eL, gamma)
            self.term = F * valid
            self.e_term = (dF + (10 + 4 * gamma) * U32 * Fhi) * valid
            self.fac = wt * Fp                                          # w_t F'(L)
            self.e_fac = wt * (dFp + (16 + 4 * gamma) * U32 * Fphi)     # its allowance
            self.D = float(target.numel())
        else:
            self.term = wt * nll
            self.e_term = (wt * e_nll + (U32 * wt * nll if kind == "wce" else 0)) * valid
            self.fac, self.e_fac = wt, torch.zeros_like(wt)
            self.D = float(wt.sum())
        n = int(valid.sum())
        self.sum = float(self.term.sum())
        self.e_sum = float(self.e_term.sum()) + max(n, 1) * 2.0 ** -53 * float(self.term.abs().sum())
        if not mean:
            self.g = 1.0
        elif kind == "ce":
            self.g = 1.0 / max(self.D, 1.0)
        else:
            self.g = 1.0 / self.D if self.D > 0 else 0.0
        self.loss = self.sum * self.g

    def check_accum(self, case, accum):
        """accum = fp64 [2] (loss sum, denominator).  Returns the usage of accum[0]."""
        a = accum.detach().cpu().double()
        check_exact(case, "accum[1] (denominator)", a[1:2], torch.tensor([self.D], dtype=torch.float64), ("i",))
        err = abs(float(a[0]) - self.sum)
        u = err / self.e_sum if self.e_sum > 0 else (math.inf if err > 0 else 0.0)
        if not u <= 1:
            raise AssertionError(f"{case}: accum[0] = {float(a[0]):.17g}, ref {self.sum:.17g}, bound {self.e_sum:.3g}, "
                                 f"usage {u:.3g}")
        return u

    def check_loss(self, case, loss):
        got = float(loss)
        e = self.e_sum * abs(self.g) + 2 * U32 * abs(self.loss)
        err = abs(got - self.loss)
        u = err / e if e > 0 else (math.inf if err > 0 else 0.0)
        if not u <= 1:
            raise AssertionError(f"{case}: loss = {got:.9g}, ref {self.loss:.9g}, bound {e:.3g}, usage {u:.3g}")
        return u

    def grad_bound(self, gscale=1.0, cpu=True):
        """Bound of dlogits [N, C, H, W] for an upstream gscale: ref = G w_t F'(L) (p_c - [c = t]), 0 at ignored pixels.
        cpu=False keeps ref and acc on the logits' device (the fused paths transform them further)."""
        sm = self.sm
        C = sm.z.shape[1]
        G = float(gscale) * self.g
        onehot = torch.nn.functional.one_hot(self.t, C).permute(0, 3, 1, 2).double()
        pd = sm.p - onehot
        fac = (G * self.fac * self.valid).unsqueeze(1)
        efac = (abs(G) * self.e_fac * self.valid).unsqueeze(1)
        ref = fac * pd
        acc = fac.abs() * (sm.ep + U32 * pd.abs()) + efac * pd.abs() + 3 * U32 * ref.abs() + SUB
        if not cpu:
            return ref, acc
        return Bound(ref.cpu(), torch.zeros_like(ref).cpu(), acc.cpu(), NAMES)


# ------------------------------------------------------------------------------------------------ Dice
def dice_fixup(target, ignore=255):
    """utils/losses.py:40-42: ignored labels become target.min() unless ignore lies in range(min, max)."""
    t = target.clone()
    if ignore not in range(int(t.min()), int(t.max())) and bool((t == ignore).any()):
        t[t == ignore] = t.min()
    return t


class DiceRef:
    """DiceLoss on a fixed-up target (every label in [0, C))."""

    def __init__(self, z, target, smooth=1.0):
        self.sm = sm = Softmax(z)
        C = sm.z.shape[1]
        t = target
        assert bool(((t >= 0) & (t < C)).all()), "Dice needs the fixed-up target"
        self.t = t
        pt = sm.p.gather(1, t.unsqueeze(1)).squeeze(1)
        ept = sm.ep.gather(1, t.unsqueeze(1)).squeeze(1)
        n = t.numel()
        self.npix = float(n)
        self.I = float(pt.sum())
        self.e_I = float(ept.sum()) + n * 2.0 ** -53 * self.I
        self.smooth = float(torch.tensor(smooth, dtype=torch.float32))
        self.D = float(sm.p.sum()) + n + self.smooth
        self.loss = 1 - (2 * self.I + self.smooth) / self.D
        self.e_loss = (2 * self.e_I + (2 * self.I + self.smooth) * n * (C + K_P) * U32 / self.D) / self.D + 2 * U32
        self.pt, self.ept = pt, ept

    def check_fwd(self, case, accum, loss):
        a = accum.detach().cpu().double()
        check_exact(case, "accum[1] (pixels)", a[1:2], torch.tensor([self.npix], dtype=torch.float64), ("i",))
        uI = abs(float(a[0]) - self.I) / self.e_I
        if not uI <= 1:
            raise AssertionError(f"{case}: dice accum[0] = {float(a[0]):.17g}, ref {self.I:.17g}, usage {uI:.3g}")
        ul = abs(float(loss) - self.loss) / self.e_loss
        if not ul <= 1:
            raise AssertionError(f"{case}: dice loss = {float(loss):.9g}, ref {self.loss:.9g}, usage {ul:.3g}")
        return max(uI, ul)

    def grad_bound(self, gscale=1.0, beta=0.0, old=None):
        sm = self.sm
        C = sm.z.shape[1]
        Dk = 2 * self.npix + self.smooth
        G = -2.0 * float(gscale) / Dk
        onehot = torch.nn.functional.one_hot(self.t, C).permute(0, 3, 1, 2).double()
        pt, ept = self.pt.unsqueeze(1), self.ept.unsqueeze(1)
        q = onehot - sm.p
        v = G * pt * q
        acc = abs(G) * (ept * q.abs() + pt * (sm.ep + U32 * q.abs())) + 4 * U32 * v.abs() + SUB
        ref = v
        if beta != 0.0:
            o = old.to(v.device).double()
            ref = beta * o + v
            acc = acc + 2 * U32 * (beta * o).abs() + U32 * ref.abs()
        return Bound(ref.cpu(), torch.zeros_like(ref).cpu(), acc.cpu(), NAMES)


# ------------------------------------------------------------------------------------------------ Lovász
class LovaszRef:
    """Lovász-softmax (classes='present', per_image=False) of NCHW fp32-exact logits; see the module docstring."""

    def __init__(self, z, target, ignore, tie_order=False):
        sm = Softmax(z)
        N, C, H, W = sm.z.shape
        dev = sm.z.device
        flat_p = sm.p.permute(0, 2, 3, 1).reshape(-1, C)
        flat_ep = sm.ep.permute(0, 2, 3, 1).reshape(-1, C)
        lab = target.reshape(-1)
        valid = lab != ignore
        vidx = valid.nonzero().flatten()
        p, ep, lv = flat_p[vidx], flat_ep[vidx], lab[vidx]
        P = vidx.numel()
        present = [c for c in range(C) if P and bool((lv == c).any())]
        self.P, self.present, self.C = P, present, C
        g_ref = torch.zeros(P, C, dtype=torch.float64, device=dev)
        g_rad = torch.zeros(P, C, dtype=torch.float64, device=dev)
        self.class_loss, self.class_bound = [], []
        self.pure_tie_clusters = 0
        for c in present:
            fg = (lv == c)
            fgd = fg.double()
            e = (fgd - p[:, c]).abs()
            delta = ep[:, c] + U32 * e * fgd
            es, order = torch.sort(e, descending=True, stable=True)
            ds, fs = delta[order], fg[order]
            Gc = float(fgd.sum())
            cf_prev = torch.cumsum(fs.double(), 0) - fs.double()
            rank = torch.arange(P, dtype=torch.float64, device=dev)
            cb_prev = rank - cf_prev
            d_fg = 1.0 / (Gc + cb_prev)
            d_bg = (Gc - cf_prev) / ((Gc + cb_prev) * (Gc + cb_prev + 1))
            d = torch.where(fs, d_fg, d_bg)
            # clusters
            lo, hi = es - ds, es + ds
            pm = torch.cummin(lo, 0).values
            sx = torch.flip(torch.cummax(torch.flip(hi, [0]), 0).values, [0])
            brk = pm[:-1] > sx[1:]
            cid = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(brk.long(), 0)])
            ncl = int(cid[-1]) + 1 if P else 0
            start = torch.zeros(ncl, dtype=torch.int64, device=dev).scatter_reduce(
                0, cid, torch.arange(P, device=dev), "amin", include_self=False)
            nf = torch.zeros(ncl, dtype=torch.float64, device=dev).index_add_(0, cid, fs.double())
            cnt = torch.zeros(ncl, dtype=torch.float64, device=dev).index_add_(0, cid, torch.ones_like(es))
            emax = torch.full((ncl,), -1.0, dtype=torch.float64, device=dev).scatter_reduce(0, cid, es, "amax")
            emin = torch.full((ncl,), 2.0, dtype=torch.float64, device=dev).scatter_reduce(0, cid, es, "amin")
            F0 = cf_prev[start[cid]]
            B0 = start[cid].double() - F0
            nfm, nbm = nf[cid], cnt[cid] - nf[cid]
            fg_lo, fg_hi = 1.0 / (Gc + B0 + nbm), 1.0 / (Gc + B0)
            bg_lo = (Gc - F0 - nfm) / ((Gc + B0 + nbm - 1).clamp_min(1) * (Gc + B0 + nbm))
            bg_hi = (Gc - F0) / ((Gc + B0) * (Gc + B0 + 1))
            dlo, dhi = torch.where(fs, fg_lo, bg_lo), torch.where(fs, fg_hi, bg_hi)
            if tie_order:
                pure = (emax == emin)[cid]
                self.pure_tie_clusters += int(((emax == emin) & (cnt > 1)).sum())
                dlo, dhi = torch.where(pure, d, dlo), torch.where(pure, d, dhi)
            rad = torch.maximum((dhi - d).abs(), (d - dlo).abs()) + D_ROUND * U32
            # |fg - p| has no derivative at 0: where the error may round to 0 the gradient may be 0 (ATen) or +-d
            rad = torch.where(es <= ds, torch.maximum(rad, dhi + D_ROUND * U32), rad)
            sign = torch.where(fs, -1.0, 1.0)
            g_ref[order, c] = sign * d
            g_rad[order, c] = rad
            self.class_loss.append(float((es * d).sum()))
            self.class_bound.append(float(ds.max()) + 4 * U32)
        n = max(len(present), 1)
        self.loss = sum(self.class_loss) / n
        self.e_loss = sum(self.class_bound) / n + U32 * abs(self.loss)
        # softmax Jacobian
        pres = torch.zeros(C, dtype=torch.bool, device=dev)
        pres[present] = True
        pp = p * pres
        dot = (pp * g_ref).sum(1, keepdim=True)
        ref = p * (g_ref - dot) / n
        mag = (pp * g_ref.abs()).sum(1, keepdim=True)
        acc = (p * (g_rad + (pp * g_rad).sum(1, keepdim=True)) + ep * (g_ref - dot).abs()
               + p * (ep * pres * g_ref.abs()).sum(1, keepdim=True) + (C + 4) * U32 * p * (g_ref.abs() + mag)) / n + SUB
        full_ref = torch.zeros(N * H * W, C, dtype=torch.float64, device=dev)
        full_acc = torch.zeros_like(full_ref)
        full_ref[vidx] = ref
        full_acc[vidx] = acc
        to_nchw = lambda t: t.view(N, H, W, C).permute(0, 3, 1, 2).cpu()  # noqa: E731
        self.grad = Bound(to_nchw(full_ref), torch.zeros(N, C, H, W, dtype=torch.float64), to_nchw(full_acc), NAMES)

    def check_loss(self, case, loss):
        err = abs(float(loss) - self.loss)
        u = err / self.e_loss
        if not u <= 1:
            raise AssertionError(f"{case}: lovasz loss = {float(loss):.9g}, ref {self.loss:.9g}, bound {self.e_loss:.3g}, "
                                 f"usage {u:.3g}")
        return u


# ------------------------------------------------------------------------------------------------ fused upsample
def rscale(inp, out, ac):
    """seg_loss.cu's rscale: the fp32 source-index scale."""
    f = torch.float32
    if ac:
        return float(torch.tensor(float(inp - 1), dtype=f) / torch.tensor(float(out - 1), dtype=f)) if out > 1 else 0.0
    return float(torch.tensor(float(inp), dtype=f) / torch.tensor(float(out), dtype=f))


def patch_for(inp, out, ac, tile):
    """Mirror of patch_for: low-res rows touched by `tile` consecutive output rows (fp32 ceilf(scale (tile - 1)) + 3)."""
    sc = torch.tensor(rscale(inp, out, ac), dtype=torch.float32) * torch.tensor(float(tile - 1), dtype=torch.float32)
    return min(math.ceil(float(sc)) + 3, inp + 1)


def upsample_schedule(Hi, Wi, Ho, Wo, C, ac, metrics=True):
    """Mirror of upsample_ce_fwd / upsample_ce_bwd's host checks: the forward's 32 x 32 tile and its patch (<= 200 KB of
    shared memory with the counters), the backward's tile 32, or 16 when the 32-tile patch's 12 B per element do not
    fit in 227 KB."""
    fp = max(patch_for(Hi, Ho, ac, 32), patch_for(Wi, Wo, ac, 32))
    fwd_smem = fp * fp * C * 4 + ((3 * C + 2) * 4 if metrics else 0)

    def bp(t):
        return max(patch_for(Hi, Ho, ac, t), patch_for(Wi, Wo, ac, t))

    tile = 32 if bp(32) ** 2 * C * 12 <= 227 * 1024 else 16
    bwd_smem = bp(tile) ** 2 * C * 12
    return {"fwd_patch": fp, "fwd_smem": fwd_smem, "fwd_ok": C <= FUSED_MAXC and fwd_smem <= 200 * 1024,
            "bwd_tile": tile, "bwd_patch": bp(tile), "bwd_smem": bwd_smem,
            "bwd_ok": C <= FUSED_MAXC and bwd_smem <= 227 * 1024,
            "last_tile_rows": Ho - (-(-Ho // tile) - 1) * tile}


def grad_scale(kind, gscale, D, mean, weight, gamma, sh, sw, Ho, Wo):
    """Mirror of ce_grad_scale(loss_grad_bound(loss_grad_g(...))): 2^(61 - e) with e the binary exponent of
    |g| max(w) (1 + gamma) (2 / sh + 2)(2 / sw + 2)."""
    f = torch.float32
    gs = torch.tensor(gscale, dtype=f)
    if kind == "ce":
        g = float(gs / torch.tensor(max(D, 1.0), dtype=f))
    elif not mean:
        g = float(gs)
    else:
        g = float(torch.tensor(float(gs) / D, dtype=f)) if D > 0 else 0.0
    gmax = g
    if kind != "ce":
        wmax = 1.0 if weight is None else max(0.0, float(weight.float().max()))
        gmax = g * wmax * ((1.0 + float(torch.tensor(gamma, dtype=f))) if kind == "focal" else 1.0)
    ry = 2.0 / sh if sh > 0 else float(Ho)
    rx = 2.0 / sw if sw > 0 else float(Wo)
    _, e = math.frexp(abs(gmax) * (ry + 2.0) * (rx + 2.0))
    return 2.0 ** (61 - e)


def _tap_counts(inp, out, ac):
    i0, i1, _, _ = lerp_axis(inp, out, ac)
    return (torch.bincount(i0, minlength=inp) + torch.bincount(i1, minlength=inp)).double()


class UpsampleRef:
    """The fused bilinear upsample + loss of NHWC fp32 low-res logits lo [N, Hi, Wi, C] to target's size.

    Forward: the interpolated logits x = Ay lo Ax^T with the kernel's fp32 lambdas (elementwise_check.lerp_matrix), each
    charged 4 u32 sum |w lo| (two lerps of two products each, fused or not), which LossRef propagates through the
    softmax.  Backward: dlo is the transpose of that interpolation applied to the per-pixel gradient; each contribution
    (fp32 lambda products times the fp32 per-pixel gradient) rounds twice and to the fixed-point quantum
    1 / (2 scale) of grad_scale; the result rounds once to fp32.  The (taps + 2) u32 sum |w g| of
    elementwise_check.bilinear_bwd_bound is charged on top, so that ATen's float32 accumulation is accepted too."""

    def __init__(self, lo, target, ac, ignore, kind, weight=None, gamma=0.0, mean=True):
        lo = lo.double()
        N, Hi, Wi, C = lo.shape
        Ho, Wo = target.shape[1:]
        dev = lo.device
        self.ac, self.shape, self.kind, self.weight, self.gamma, self.mean = ac, (N, Hi, Wi, C, Ho, Wo), kind, weight, gamma, mean
        self.Ay, self.Ax = lerp_matrix(Hi, Ho, ac).to(dev), lerp_matrix(Wi, Wo, ac).to(dev)
        self.x = torch.einsum("oh,nhwc,pw->ncop", self.Ay, lo, self.Ax)
        self.ev = 4 * U32 * torch.einsum("oh,nhwc,pw->ncop", self.Ay.abs(), lo.abs(), self.Ax.abs())
        self.loss = LossRef(self.x, target, ignore, kind, weight, gamma, mean, ev=self.ev)

    def grad_out(self, gscale=1.0):
        """Per-output-pixel gradient (ref, allowance), NCHW [N, C, Ho, Wo], on the logits' device."""
        return self.loss.grad_bound(gscale, cpu=False)

    def dlo_bound(self, gscale=1.0, Ay=None):
        N, Hi, Wi, C, Ho, Wo = self.shape
        Ay = self.Ay if Ay is None else Ay
        ref_o, acc_o = self.grad_out(gscale)
        ref = torch.einsum("oh,ncop,pw->nhwc", Ay, ref_o, self.Ax)
        mag = torch.einsum("oh,ncop,pw->nhwc", Ay.abs(), ref_o.abs(), self.Ax.abs())
        acc_t = torch.einsum("oh,ncop,pw->nhwc", Ay.abs(), acc_o, self.Ax.abs())
        taps = ((Ay != 0).sum(0).view(Hi, 1) * (self.Ax != 0).sum(0).view(1, Wi)).double().view(1, Hi, Wi, 1)
        contrib = (_tap_counts(Hi, Ho, self.ac).view(Hi, 1) * _tap_counts(Wi, Wo, self.ac).view(1, Wi)).view(1, Hi, Wi, 1)
        scale = grad_scale(self.kind, gscale, self.loss.D, self.mean, self.weight, self.gamma,
                           rscale(Hi, Ho, self.ac), rscale(Wi, Wo, self.ac), Ho, Wo)
        acc = acc_t + (taps + 2) * U32 * mag + 0.5 / scale * contrib.to(ref.device) + U32 * ref.abs() + SUB
        return Bound(ref.cpu(), torch.zeros_like(ref).cpu(), acc.cpu(), ("n", "h", "w", "c"))


def check_argmax(case, got, x, ev, show=8):
    """got [N, Ho, Wo]: the kernel's arg-max of its fp32 logits.  Where the float64 maximum is tied exactly (planted
    equal sources) it must be the first maximum; otherwise it may be any class within the two values' allowances of
    the maximum.  Returns the number of pixels that took a legitimate runner-up."""
    g = got.to(x.device).long().unsqueeze(1)
    top = x.amax(1)
    first = first_argmax(x).unsqueeze(1)
    xa, ea = x.gather(1, g).squeeze(1), ev.gather(1, g).squeeze(1)
    et = ev.gather(1, first).squeeze(1)
    ok = ((xa == top) & (g.squeeze(1) == first.squeeze(1))) | ((xa < top) & (xa >= top - ea - et))
    bad = (~ok).nonzero()
    if bad.shape[0]:
        lines = [f"  (n, h, w)={tuple(ix)}: got {int(g[ix[0], 0, ix[1], ix[2]])}, first max {int(first[ix[0], 0, ix[1], ix[2]])}"
                 for ix in bad[:show].tolist()]
        raise AssertionError(f"{case}: arg-max: {bad.shape[0]} pixel(s) wrong\n" + "\n".join(lines))
    return int((g.squeeze(1) != first.squeeze(1)).sum())


# ------------------------------------------------------------------------------------------------ fused shuffle
def shuffle_logits(lo, r, C):
    """The NCHW logits [N, C, h r, w r] the shuffle loss reads in place from NHWC lo [N, h, w, >= r^2 C]: class c of
    pixel (y r + i, x r + j) is channel c r^2 + i r + j of low-res pixel (y, x) (nn.PixelShuffle(r))."""
    return F.pixel_shuffle(lo[..., :r * r * C].permute(0, 3, 1, 2), r)


class ShuffleRef:
    """The fused pixel-shuffle + loss of bf16 NHWC lo: LossRef of the exact shuffled logits; dx [N, h, w, r^2 C] is the
    per-pixel gradient unshuffled, each element written once as the bf16 rounding of its fp32 value."""

    def __init__(self, lo, r, C, target, ignore, kind, weight=None, gamma=0.0, mean=True):
        self.r = r
        self.loss = LossRef(shuffle_logits(lo.double(), r, C), target, ignore, kind, weight, gamma, mean)

    def dx_bound(self, gscale=1.0):
        ref, acc = self.loss.grad_bound(gscale, cpu=False)
        un = lambda t: F.pixel_unshuffle(t, self.r).permute(0, 2, 3, 1).cpu()  # noqa: E731
        return bound(un(ref), un(acc), True, ("n", "h", "w", "ch"))


def check_pad(case, dx, width):
    """The pad lanes [width, pitch) of a bf16 gradient [rows, pitch] must be exactly zero."""
    pad = dx.reshape(-1, dx.shape[-1])[:, width:].float().cpu()
    bad = (pad != 0).nonzero()
    if bad.shape[0]:
        raise AssertionError(f"{case}: {bad.shape[0]} pad lane(s) not zero, first (row, lane) "
                             f"{tuple(bad[0].tolist())} = {pad[tuple(bad[0].tolist())].item()}")


# ------------------------------------------------------------------------------------------------ metrics
def metrics_ref(z, target, K):
    """eval_metrics counters [2 + 3K] (correct, labeled, inter[K], pred[K], lab[K]) with the first-maximum arg-max."""
    return counters_from_map(first_argmax(z), target, K)


def counters_from_map(pred, target, K):
    """The same counters from a given arg-max map (the fused kernels count from the map they write)."""
    pred = pred.reshape(-1).cpu().long()
    t = target.reshape(-1).cpu()
    lab = (t >= 0) & (t < K)
    pl, tl = pred[lab], t[lab]
    corr = pl == tl
    out = torch.zeros(2 + 3 * K, dtype=torch.int64)
    out[0] = int(corr.sum())
    out[1] = int(lab.sum())
    out[2:2 + K] = torch.bincount(tl[corr], minlength=K)[:K]
    out[2 + K:2 + 2 * K] = torch.bincount(pl[pl < K], minlength=K)[:K]
    out[2 + 2 * K:] = torch.bincount(tl, minlength=K)[:K]
    return out


# ------------------------------------------------------------------------------------------------ operands
def logits(N, C, H, W, seed, sat=False, top=6):
    """fp32 logits with per-pixel scales 2^-9 .. 2^top (near-uniform and near-one-hot softmaxes); sat: a block of
    +-1e3."""
    g = torch.Generator().manual_seed(seed)
    s = 2.0 ** torch.randint(-9, top + 1, (N, 1, H, W), generator=g).float()
    z = torch.randn(N, C, H, W, generator=g) * s
    if sat:
        z[:, :, : H // 4, : W // 4] = torch.where(torch.rand(N, C, H // 4, W // 4, generator=g) < 0.5, 1e3, -1e3)
    return z


def labels(N, H, W, C, seed, ignore=255, frac=0.1):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, C, (N, H, W), generator=g)
    return torch.where(torch.rand(N, H, W, generator=g) < frac, torch.full_like(t, ignore), t)


def weights(C, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(C, generator=g) * 2
    w[::5] = 0
    return w


def lovasz_case(N=1, C=8, H=512, W=512, seed=11, rare=3, top=6):
    z = logits(N, C, H, W, seed, top=top)
    t = labels(N, H, W, C, seed + 1)
    t[t == 0] = 1
    g = torch.Generator().manual_seed(seed + 2)
    idx = torch.randperm(N * H * W, generator=g)[:rare]
    t.view(-1)[idx] = 0  # class 0 is rare: its Jaccard steps are large
    return z, t


def tie_case(N=1, C=8, H=256, W=256, seed=31, groups=2000, size=4):
    """Groups of pixels with bit-identical logit vectors and labels, spread over the image, each confident in a rare
    class it is not labelled with.  The other pixels' logits are small, so the groups rank at the top of that class,
    where the Jaccard steps are large."""
    z, t = lovasz_case(N, C, H, W, seed, top=0)
    g = torch.Generator().manual_seed(seed + 5)
    perm = torch.randperm(N * H * W, generator=g)[:groups * size].view(groups, size)
    zf = z.permute(0, 2, 3, 1).reshape(-1, C)
    tf = t.view(-1)
    for k in range(groups):
        v = torch.randn(C, generator=g)
        v[0] += 4 + 4 * torch.rand(1, generator=g).item()
        zf[perm[k]] = v
        tf[perm[k]] = 1 + k % (C - 1)
    z = zf.view(N, H, W, C).permute(0, 3, 1, 2).contiguous()
    return z, t
