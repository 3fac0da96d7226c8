"""References, bounds and schedule mirrors for the parameter-path kernels (seg_elementwise.cu): the batched weight
packing and weight-gradient unpacking of `train.WeightTables`, the single-tensor `seg_pack_weight` / `seg_unpack_wgrad`,
and the multi-tensor SGD kernel of `seg_sgd_step` / `seg_sgd_step_dev`.

Pure torch / numpy; it imports nothing from the library, so its own tests run without a GPU (test_param_check_cpu.py)
and the GPU sweep (test_param_conformance_gpu.py) feeds it what the kernels wrote.  The references work on any device
in float64 from the exact fp32 inputs.

Packing is exact: bf16 round-to-nearest-even of the fp32 bit pattern, done here in integer arithmetic.  Unpacking is
exact with beta = 0; with beta != 0 each element is `beta * old + v` in fp32, at most two roundings:

    |got - ref| <= gamma(2) (|beta old| + |v|)

SGD (torch.optim.SGD with dampening 0, no Nesterov; s = grad_scale, lambda = weight decay, mu = momentum, eta = lr):

    d = g s + lambda p,   m = d (first step or mu = 0) else mu b + d,   p' = p - eta m
    |m - m64|  <= gamma(3) M,            M = |g s| + |lambda p| + |mu b|
    |p' - p'64| <= gamma(5) (|p| + eta M)

with gamma(n) = n u / (1 - n u), u = 2^-24.  Both hold whether or not the compiler contracts the products into FMAs.
mu = 0 leaves the buffer untouched and eta = 0 the parameter, bit for bit.
"""
import math

import numpy as np
import torch

U32 = 2.0 ** -24
THREADS = 256
BATCHED_BLOCKS = 48                         # pack_weights_batched / unpack_wgrads_batched: grid (48, rows)
BATCHED_STRIDE = BATCHED_BLOCKS * THREADS   # 12288 elements per grid-stride pass of one table row
SGD_BLOCKS = 64                             # sgd_kernel: grid (64, tensors)
SGD_STRIDE = SGD_BLOCKS * THREADS           # 16384
SINGLE_BLOCKS_PER_SM = 8                    # grid_for(total, 256) of seg_pack_weight / seg_unpack_wgrad
MAX_ROWS = 65535                            # gridDim.y limit: table rows / tensors per launch

# mirror of train.WeightTables's entry (PackEntry in seg_elementwise.cu)
PACK_DTYPE = np.dtype([("oihw", "<u8"), ("packed", "<u8"), ("K", "<i4"), ("C", "<i4"), ("R", "<i4"), ("S", "<i4"),
                       ("Cpad", "<i4"), ("explicit", "<i4"), ("start", "<i8")])


def gamma(n):
    return n * U32 / (1 - n * U32)


# ------------------------------------------------------------------------------------------------ schedule mirrors
def batched_passes(count):
    """Grid-stride passes the busiest thread of one batched pack / unpack row makes over `count` elements."""
    return max(1, -(-count // BATCHED_STRIDE))


def sgd_passes(n):
    return max(1, -(-n // SGD_STRIDE))


def single_grid(total, sms):
    """Blocks of grid_for(total, 256): one element per thread until the cap of SMs * 8 blocks."""
    return max(1, min(-(-total // THREADS), sms * SINGLE_BLOCKS_PER_SM))


def single_cap(sms):
    """Elements one pass of the capped single pack / unpack grid covers."""
    return sms * SINGLE_BLOCKS_PER_SM * THREADS


def single_passes(total, sms):
    return max(1, -(-total // (single_grid(total, sms) * THREADS)))


# ------------------------------------------------------------------------------------------------ packing
def kpad_for(R, S, C):
    return (R * S * C + 7) // 8 * 8


def bf16_bits(x):
    """bf16 round-to-nearest-even of fp32 `x`, as int16 bit patterns, in integer arithmetic on the fp32 bits (finite
    inputs; a carry out of the largest finite magnitudes gives the infinity, as the hardware conversion does)."""
    assert x.dtype == torch.float32
    assert bool(torch.isfinite(x).all()), "bf16_bits: finite inputs only"
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    r = torch.where(r >= 0x8000, r - 0x10000, r)
    return r.to(torch.int16)


def packed_shape(K, C, R, S, explicit, cpad=None):
    if explicit:
        return (1, K, kpad_for(R, S, C) if cpad is None else cpad)
    return (R * S, K, C if cpad is None else cpad)


def pack_ref(w_oihw, explicit, kpad=None):
    """Expected bf16 bits (int16) of the packed weight, for w [..., K, C, R, S] (leading batch dims allowed).
    Normal rows: [R*S][K][Cpad] (kpad = Cpad, default C).  Explicit rows: [1][K][Kpad], column (r*S + s)*C + c, default
    Kpad = R*S*C rounded up to 8.  Pad columns are +0.0 (bits 0x0000)."""
    *lead, K, C, R, S = w_oihw.shape
    if explicit:
        kp = kpad_for(R, S, C) if kpad is None else kpad
        assert kp >= R * S * C
        src = w_oihw.permute(*range(len(lead)), -4, -2, -1, -3).reshape(*lead, 1, K, R * S * C)
    else:
        kp = C if kpad is None else kpad
        assert kp >= C
        src = w_oihw.permute(*range(len(lead)), -2, -1, -4, -3).reshape(*lead, R * S, K, C)
    bits = bf16_bits(src.float())
    if kp > src.shape[-1]:
        pad = torch.zeros(*bits.shape[:-1], kp - src.shape[-1], dtype=torch.int16, device=bits.device)
        bits = torch.cat([bits, pad], -1)
    return bits


def check_pack(case, got_bits, want_bits, show=8):
    """Bit-exact comparison of int16 patterns; reports the first differing coordinates ([tap][k][column])."""
    got, want = got_bits.detach().cpu(), want_bits.detach().cpu()
    assert got.shape == want.shape, (case, tuple(got.shape), tuple(want.shape))
    bad = (got != want).nonzero()
    if bad.shape[0]:
        lines = [f"  {tuple(ix)}: got=0x{int(got[tuple(ix)]) & 0xFFFF:04x} want=0x{int(want[tuple(ix)]) & 0xFFFF:04x}"
                 for ix in bad[:show].tolist()]
        raise AssertionError(f"{case}: pack: {bad.shape[0]} element(s) differ\n" + "\n".join(lines))


# ------------------------------------------------------------------------------------------------ unpacking
def unpacked_view(packed, K, C, R, S, explicit):
    """The OIHW [..., K, C, R, S] view of a packed [..., taps, K, Cpad] gradient; pad columns are not read."""
    *lead, T, Kk, cpad = packed.shape
    assert Kk == K
    if explicit:
        assert T == 1
        v = packed[..., 0, :, :R * S * C].reshape(*lead, K, R, S, C)
        return v.permute(*range(len(lead)), -4, -1, -3, -2)
    assert T == R * S
    v = packed[..., :C].reshape(*lead, R, S, K, C)
    return v.permute(*range(len(lead)), -2, -1, -4, -3)


def unpack_ref(packed, K, C, R, S, Cpad, explicit, beta=0.0, old=None):
    """(ref, bound) in float64 OIHW for `g = beta * old + packed` (beta = 0: old is not read; bound 0 = exact)."""
    assert packed.shape[-1] == Cpad
    v = unpacked_view(packed, K, C, R, S, explicit).double()
    if beta == 0.0:
        return v, torch.zeros_like(v)
    bo = float(np.float32(beta)) * old.double()
    return bo + v, gamma(2) * (bo.abs() + v.abs())


def _bits32(t):
    return t.contiguous().view(torch.int32)


def check_bounded(case, what, got, ref, bound, show=8):
    """Every element of fp32 `got` within `bound` of `ref`; where the bound is 0 the fp32 bits must match ref's (exact
    results, NaN or not).  Returns the largest bound usage (|err| / bound, 0 where exact)."""
    got = got.detach()
    ref, bound = ref.to(got.device), bound.to(got.device)
    assert got.shape == ref.shape, (case, what, tuple(got.shape), tuple(ref.shape))
    g64 = got.double()
    err = (g64 - ref).abs()
    exact = bound == 0
    usage_t = torch.where(exact, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    exact_bad = exact & (_bits32(got) != _bits32(ref.float()))
    usage_t = torch.where(exact_bad | torch.isnan(g64) & ~exact, torch.full_like(usage_t, math.inf), usage_t)
    usage = usage_t.max().item() if usage_t.numel() else 0.0
    bad = (usage_t > 1).nonzero()
    if bad.shape[0]:
        lines = []
        for ix in bad[:show].tolist():
            t = tuple(ix)
            lines.append(f"  {t}: got={g64[t].item():.9g} ref={ref[t].item():.9g} bound={bound[t].item():.3g}")
        raise AssertionError(f"{case}: {what}: {bad.shape[0]} element(s) over the bound, bound usage {usage:.3g}\n"
                             + "\n".join(lines))
    return usage


# ------------------------------------------------------------------------------------------------ SGD
class SgdRef:
    """p, m: float64 results; bp, bm: their bounds; keep_buf / keep_p: the buffer (mu = 0) / parameter (eta = 0) must
    come back bit for bit."""

    def __init__(self, p, m, bp, bm, keep_buf, keep_p):
        self.p, self.m, self.bp, self.bm, self.keep_buf, self.keep_p = p, m, bp, bm, keep_buf, keep_p


def f32(x):
    return float(np.float32(x))


def sgd_ref(p, g, buf, lr, mom, wd, gscale, first_step):
    """Float64 reference of one sgd_kernel tensor from its exact fp32 inputs.  The scalars are rounded to the fp32 values
    the kernel receives (e.g. float32(1/3) for grad_scale)."""
    lr, mom, wd, gscale = f32(lr), f32(mom), f32(wd), f32(gscale)
    p64, g64 = p.double(), g.double()
    gs, lp = g64 * gscale, wd * p64
    use_b = mom != 0.0 and not first_step
    mb = mom * buf.double() if use_b else torch.zeros_like(p64)
    m = gs + lp + mb
    mag = gs.abs() + lp.abs() + mb.abs()
    pn = p64 - lr * m
    bm = gamma(3) * mag
    bp = gamma(5) * (p64.abs() + lr * mag)
    return SgdRef(pn, m, bp, bm, mom == 0.0, lr == 0.0)


def check_sgd(case, r, p_new, buf_new, p_old, buf_old):
    """Checks one tensor's new parameter and momentum buffer; returns the larger bound usage."""
    if r.keep_p:
        assert torch.equal(_bits32(p_new), _bits32(p_old.to(p_new.device))), f"{case}: lr = 0 changed the parameter"
        up = 0.0
    else:
        up = check_bounded(case, "param", p_new, r.p, r.bp)
    if r.keep_buf:
        assert torch.equal(_bits32(buf_new), _bits32(buf_old.to(buf_new.device))), \
            f"{case}: momentum 0 wrote the momentum buffer"
        um = 0.0
    else:
        um = check_bounded(case, "momentum", buf_new, r.m, r.bm)
    return max(up, um)


# ------------------------------------------------------------------------------------------------ fp32 emulations
def _rn(x):
    return x.float()


def sgd_emulate(p, g, buf, lr, mom, wd, gscale, first_step, fma):
    """sgd_kernel in fp32 on the CPU: every operation rounded to fp32 (fma=False), or the products contracted into
    fused multiply-adds the way nvcc may contract them (fma=True; the float64 sum of an exact product is rounded once).
    Returns (p', buffer')."""
    lr, mom, wd, gscale = (torch.tensor(f32(v), dtype=torch.float32) for v in (lr, mom, wd, gscale))
    if fma:
        d = _rn(g.double() * gscale.double() + _rn(wd * p).double())
    else:
        d = _rn(_rn(g * gscale) + _rn(wd * p))
    b = buf.clone()
    if float(mom) != 0.0:
        if first_step:
            m = d
        elif fma:
            m = _rn(mom.double() * buf.double() + d.double())
        else:
            m = _rn(_rn(mom * buf) + d)
        b = m
        d = m
    if fma:
        pn = _rn(p.double() - lr.double() * d.double())
    else:
        pn = _rn(p - _rn(lr * d))
    return pn, b


def unpack_emulate(packed, K, C, R, S, explicit, beta, old, fma):
    v = unpacked_view(packed, K, C, R, S, explicit).float()
    if beta == 0.0:
        return v.clone(memory_format=torch.contiguous_format)
    b = torch.tensor(f32(beta), dtype=torch.float32)
    if fma:
        return _rn(b.double() * old.double() + v.double())
    return _rn(_rn(b * old) + v)


# ------------------------------------------------------------------------------------------------ tables
def build_table(rows, kind):
    """rows: (oihw_ptr, packed_ptr, K, C, R, S, Cpad, explicit) in table order; kind "pack" (start = prefix sum of packed
    elements) or "unpack" (of OIHW elements).  Returns (numpy PACK_DTYPE array, total work items)."""
    tab = np.zeros(len(rows), dtype=PACK_DTYPE)
    start = 0
    for i, (po, pp, K, C, R, S, cpad, ex) in enumerate(rows):
        tab[i] = (po, pp, K, C, R, S, cpad, int(ex), start)
        start += (K * cpad if ex else R * S * K * cpad) if kind == "pack" else K * C * R * S
    return tab, start


def spec_rows(specs, packed_bufs, dw_bufs, grad_views):
    """(pack rows, unpack rows) of a model's dense convs, from each weight's shape alone: K, C, R, S = weight.shape (a
    transposed conv's [Cin, Cout, k, k] read as OIHW), explicit im2col for C % 8 != 0 or a conv the model marks explicit,
    Kpad = R*S*C rounded up to 8.  Unpack rows only for trainable weights, in spec order."""
    pack, unpack = [], []
    for s in specs:
        w = s.m.weight
        K, C, R, S = w.shape
        ex = bool(s.explicit) or C % 8 != 0
        cpad = kpad_for(R, S, C) if ex else C
        pack.append((w.data_ptr(), packed_bufs[s].data_ptr(), K, C, R, S, cpad, ex))
        if grad_views is not None and w.requires_grad:
            unpack.append((grad_views[w].data_ptr(), dw_bufs[s].data_ptr(), K, C, R, S, cpad, ex))
    return pack, unpack
